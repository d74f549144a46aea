"""FLAME texture space on the GPU -- the drop-in for ``FlameTextureSpace`` (model/stg2_generator.py:336-421) and for
``InterpolatedTextureLoss`` (loss_functions/losses.py:127-235), SURVEY 8f.2.

``FlameTextureSpace.forward(source_img, flame_params_full)`` "steals" a UV texture from a generated image: FLAME decode
(gifb200_flame_lbs) -> projection + vertex normals -> ``gifb200_texture_steal_fwd`` (one fused pass instead of six
gathers, two scatters and a grid_sample).  Differentiable w.r.t. the image (that is where the loss's gradient flows into
the generator); the FLAME parameters are data, as in the reference."""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from ._lib import check, lib, ptr, require_cuda, stream
from .render import batch_orth_proj, vertex_adjacency, vertex_normals


class _TextureSteal(torch.autograd.Function):
    """tex (B,T,T,C) = S(src (B,H,W,C)); S is linear in src, so the backward is the adjoint kernel and the backward of
    the backward is S again (closed under differentiation like every op of this package)."""

    @staticmethod
    def forward(ctx, src, verts, normals, cam, table, want_mask):
        src, verts, cam = ops._c(src), ops._c(verts), ops._c(cam)
        require_cuda(src, verts, normals, cam)
        B, H, W, C = src.shape
        T, V = table["T"], verts.shape[1]
        tex = torch.empty(B, T, T, C, device=src.device)
        mask = torch.empty(B, T, T, dtype=torch.uint8, device=src.device) if want_mask else None
        check(lib.gifb200_texture_steal_fwd(ptr(src), ptr(verts), ptr(None if normals is None else ops._c(normals)), ptr(cam),
                                            ptr(table["texel_to_valid"]), ptr(table["vid"]), ptr(table["bary"]), ptr(tex),
                                            ptr(mask), B, H, W, C, V, T, stream()), "gifb200_texture_steal_fwd")
        ctx.save_for_backward(verts, cam)
        ctx.table, ctx.src_shape = table, (B, H, W, C)
        if want_mask:
            ctx.mark_non_differentiable(mask)
            return tex, mask
        return tex, None

    @staticmethod
    def backward(ctx, g_tex, _g_mask):
        verts, cam = ctx.saved_tensors
        return _TextureStealAdjoint.apply(g_tex, verts, cam, ctx.table, ctx.src_shape), None, None, None, None, None


class _TextureStealAdjoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, g_tex, verts, cam, table, src_shape):
        g_tex = ops._c(g_tex)
        require_cuda(g_tex)
        B, H, W, C = src_shape
        g_src = torch.empty(B, H, W, C, device=g_tex.device)
        check(lib.gifb200_texture_steal_bwd(ptr(g_tex), ptr(verts), ptr(cam), ptr(table["texel_to_valid"]), ptr(table["vid"]),
                                            ptr(table["bary"]), ptr(g_src), B, H, W, C, verts.shape[1], table["T"], stream()),
              "gifb200_texture_steal_bwd")
        ctx.save_for_backward(verts, cam)
        ctx.table = table
        return g_src

    @staticmethod
    def backward(ctx, gg):
        verts, cam = ctx.saved_tensors
        return _TextureSteal.apply(gg, verts, None, cam, ctx.table, False)[0], None, None, None, None


def texture_table(texture_data, size=256, device="cuda"):
    """Kernel-side form of the reference's table (stg2_generator.py:349-354): a dense texel -> entry map + (N,3) vertex ids
    and barycentrics."""
    valid = np.asarray(texture_data["valid_pixel_ids"]).astype(np.int64)
    ys = np.asarray(texture_data["y_coords"]).astype(np.int64)[valid]
    xs = np.asarray(texture_data["x_coords"]).astype(np.int64)[valid]
    t2v = -np.ones(size * size, dtype=np.int32)
    t2v[ys * size + xs] = np.arange(valid.size, dtype=np.int32)       # later entries win, like the reference's index_put
    return {"T": size, "texel_to_valid": torch.from_numpy(t2v).to(device),
            "vid": torch.from_numpy(np.asarray(texture_data["valid_pixel_3d_faces"]).astype(np.int32)).contiguous().to(device),
            "bary": torch.from_numpy(np.asarray(texture_data["valid_pixel_b_coords"]).astype(np.float32)).contiguous().to(device)}


class FlameTextureSpace(nn.Module):
    """model/stg2_generator.py:336-421.  ``texture_data``: the pre-computed table (x_coords, y_coords, valid_pixel_ids,
    valid_pixel_3d_faces, valid_pixel_b_coords); ``flame``: a ``gif_b200.flame.FLAME`` (the reference builds its own from
    ``constants.flame_config``, which needs the licence-gated model file)."""

    def __init__(self, texture_data, data_un_normalizer=None, flame=None, size=256):
        super().__init__()
        if flame is None:
            flame = self._flame_from_constants()
        self.texture_data = texture_data
        self.data_un_normalizer = data_un_normalizer
        self.flame = flame
        self.size = size
        self._table = None
        self._adj = None

    @staticmethod
    def _flame_from_constants():
        """The reference builds its decoder from ``constants.flame_config`` (gen.py:343-347 via gif_helper.render_utils);
        as a drop-in under the reference's tree the same config (and its licence-gated generic_model.pkl) is used."""
        import types
        try:
            import constants as cnst
        except ImportError as e:
            raise ValueError("FlameTextureSpace needs a gif_b200.flame.FLAME decoder (flame=...) when the reference's "
                             "`constants` module is not importable") from e
        from .flame import FLAME
        return FLAME(types.SimpleNamespace(**cnst.flame_config))

    def _tab(self, device):
        if self._table is None or self._table["vid"].device != device:
            self._table = texture_table(self.texture_data, self.size, device)
        return self._table

    def forward(self, source_img, flame_params_full):
        """source_img (B,C,H,W) (any layout; channels-last storage is zero-copy), flame_params_full (B,>=159) =
        [shape 100 | exp 50 | pose 6 | cam 3] -> (texture_img (B,C,T,T), texture_vis_mask (B,1,T,T) bool)."""
        if self.data_un_normalizer is not None:
            flame_params_full = self.data_un_normalizer(flame_params_full)
        p = flame_params_full.float()
        shape, exp, pose, cam = p[:, 0:100], p[:, 100:150], p[:, 150:156], p[:, 156:159].contiguous()
        with torch.no_grad():
            verts, _ = self.flame.decode_vertices(shape, exp, pose)
            trans = batch_orth_proj(verts, cam)
            trans[:, :, 1:] = -trans[:, :, 1:]
            if self._adj is None or self._adj[0].device != trans.device:
                self._adj = vertex_adjacency(self.flame.faces_tensor.to(trans.device), trans.shape[1])
            normals = vertex_normals(trans, self.flame.faces_tensor, self._adj)
        return self.compute_texture_map(source_img, verts, normals, camera_params=cam)

    def compute_texture_map(self, source_img, target_mesh_v, vertex_normals, camera_params):
        """stg2_generator.py:376-421."""
        tex, mask = _TextureSteal.apply(ops.to_nhwc(source_img), target_mesh_v, vertex_normals, camera_params,
                                        self._tab(source_img.device), True)
        return ops.to_nchw_view(tex), mask.bool()[:, None]


class InterpolatedTextureLoss:
    """loss_functions/losses.py:127-235.  The reference wires its pieces from ``constants`` (texture table, face-region
    mask image, OverLayViz renderer, all licence-gated files); here they are injected:
      flm_tex_dec            a FlameTextureSpace;
      render_condition       callable flame_batch (n,159|236) -> condition maps (n,6,256,256) in [-1,1]
                             (losses.py:186-221: rendered FLAME texture image + normal map);
      face_region_only_mask  (1,1,h,w) float tensor in [0,1] (losses.py:132-134), resized to the texture size if needed.
    """

    def __init__(self, max_images_in_batch, flm_tex_dec, render_condition, face_region_only_mask, rng=None):
        """``rng``: a numpy-RandomState-like object (default ``numpy.random``, as the reference) for the pair choice and
        the shared identity; ``rng="device"`` draws both with torch on the device instead, which keeps the whole term
        capturable in a CUDA graph (host random numbers would be frozen into the graph)."""
        self.flm_tex_dec = flm_tex_dec
        self.render_condition = render_condition
        self.face_region_only_mask = face_region_only_mask
        self.max_num = max_images_in_batch - 1
        self.pairs = np.array([(i, j) for i in range(self.max_num) for j in range(i + 1, self.max_num)])   # :141-145
        self.rng = rng if rng is not None else np.random

    def pairwise_texture_loss(self, tx1, tx2):
        """losses.py:147-159."""
        m = self.face_region_only_mask.to(tx1.device)
        if m.shape[-1] != tx1.shape[-1]:
            m = torch.nn.functional.interpolate(m, size=(tx1.shape[1], tx1.shape[2]), mode="bilinear", align_corners=False)
            self.face_region_only_mask = m
        return torch.mean(torch.sigmoid(torch.pow(tx1 - tx2, 2)) * m[0])

    def tex_sp_intrp_loss(self, flame_batch, generator, step, alpha, max_ids, normal_maps_as_cond=True,
                          use_posed_constant_input=False, rendered_flame_as_condition=True):
        """losses.py:161-176."""
        textures, tx_masks, _ = self.get_image_and_textures(alpha, flame_batch, generator, max_ids, normal_maps_as_cond,
                                                            rendered_flame_as_condition, step, use_posed_constant_input)
        if isinstance(self.rng, str):       # "device": same arithmetic, batched over the chosen pairs
            dev = textures.device
            if getattr(self, "_pairs_dev", None) is None or self._pairs_dev.device != dev:
                self._pairs_dev = torch.as_tensor(self.pairs, device=dev)      # cached: no host copy inside a graph capture
            pairs = self._pairs_dev
            sel = torch.randperm(len(self.pairs), device=dev)[:self.max_num]
            i, j = pairs[sel, 0], pairs[sel, 1]
            common = (tx_masks[j] * tx_masks[i]).to(textures.dtype)
            m = self.face_region_only_mask.to(dev)
            if m.shape[-1] != textures.shape[-1]:
                m = torch.nn.functional.interpolate(m, size=textures.shape[-2:], mode="bilinear", align_corners=False)
                self.face_region_only_mask = m
            per_pair = (torch.sigmoid(torch.pow(textures[i] * common - textures[j] * common, 2)) * m[0]).mean(dim=(1, 2, 3))
            return 16 * per_pair.sum() / sel.numel()          # len(random_pairs), losses.py:176
        sel = self.rng.choice(len(self.pairs), self.max_num, replace=False)
        loss = 0
        for i, j in self.pairs[sel]:
            common = tx_masks[j] * tx_masks[i]
            loss = loss + self.pairwise_texture_loss(textures[i] * common, textures[j] * common)
        return 16 * loss / len(sel)

    def get_image_and_textures(self, alpha, flame_batch, generator, max_ids, normal_maps_as_cond,
                               rendered_flame_as_condition, step, use_posed_constant_input):
        """losses.py:178-235: one identity for the whole (truncated) batch, one generator forward, texture stealing."""
        if flame_batch.shape[0] < self.max_num:
            # the pair table indexes textures 0..max_num-1 (losses.py:141-145); a shorter batch would be an out-of-range
            # device gather (an assert that poisons the context, or garbage under graph replay), not an IndexError
            raise ValueError(f"InterpolatedTextureLoss(max_images_in_batch={self.max_num + 1}) needs at least {self.max_num} "
                             f"interpolated label rows, got {flame_batch.shape[0]}: build it with the per-GPU batch size")
        flame_batch = flame_batch[:self.max_num, :]
        with torch.no_grad():
            cond = self.render_condition(flame_batch)
        if rendered_flame_as_condition and normal_maps_as_cond:
            gen_in = cond
        elif rendered_flame_as_condition:
            gen_in = cond[:, :3]
        elif normal_maps_as_cond:
            gen_in = cond[:, 3:]
        else:
            gen_in = flame_batch
        if isinstance(self.rng, str):
            fixed = torch.randint(0, max_ids, (1,), device=flame_batch.device).expand(flame_batch.shape[0])
        else:
            fixed = torch.ones(flame_batch.shape[0], dtype=torch.long, device=flame_batch.device) * int(self.rng.randint(0, max_ids))
        pose = flame_batch[:, 150:153] if use_posed_constant_input else None
        generated_image = generator(gen_in, pose=pose, step=step, alpha=alpha, input_indices=fixed)[-1]
        textures, tx_masks = self.flm_tex_dec(generated_image, flame_batch)
        return textures, tx_masks, generated_image
