"""Faces from FLAME parameters on the device: the chain every sampling script of the reference runs
(plots/generate_random_samples.py:156-228, plots/role_of_different_parameters.py, plots/teaser/*,
plots/voca/generate_voca_animation.py, my_utils/generate_gif.py), with nothing crossing to the host:

    1. FLAME decode, once per batch (the reference decodes twice, in position_to_given_location and in the render; shape,
       expression and pose are the same both times, so are the vertices)
    2. eye-centred camera (gif_b200.eye_centering; my_utils/eye_centering.py:35-66) written into columns 156:159
    3. the texture + normal condition (OverLayViz.get_rendered_mesh, quantised) and the "mesh" picture the scripts save
       next to each sample: the same render with a constant albedo of 0.6
    4. condition bytes -> [-1, 1] (``u8_to_unit``: for these bytes bitwise the reference's clamp(floor(.)/255, 0, 1)*2 - 1)
    5. the EMA generator at step log2(R) - 2, alpha 1
    6. image bytes as save_set_of_images writes them (``image_to_u8``: uint8(clip((clamp(x,-1,1)+1)/2, 0, 1) * 255))

``graphs=True`` captures the whole batch in one CUDA graph after one eager warm-up at the same shape; rows and identities
are copied into static buffers and one replay produces every output.  A short last batch is padded to the captured size
by repeating its last row and the extra outputs are dropped -- which is sound because no kernel on this path mixes the
samples of a batch (tests/test_sampler_gpu.py permutes a batch and checks that every output is permuted bitwise).  The
eager path pads the same way, so both compute at one batch shape and agree bitwise."""
import math

import torch

from .conditions import DECA_COLUMNS, DECA_SLICES, split_deca
from .eye_centering import eye_camera
from .flame import FLAMETex
from .image_decode import image_to_u8, u8_to_unit

# plots/generate_random_samples.py:200-201: get_rendered_mesh(..., constant_albedo=0.6).  The render works in the texture
# space's 0..255 units, so at 0.6 the quantised picture holds levels 0..2 and the saved bytes are (nearly) black -- which is
# what the reference saves; ``mesh_albedo`` picks a visible grey (e.g. 150) instead.
MESH_ALBEDO = 0.6


class FlameSampler:
    """``FlameSampler(g_running, DecaConditionRenderer(...), resolution=256).sample(rows, identity_indices)``.

    generator: a ``StyledGenerator`` conditioned on the rendered texture + normal map (the EMA generator of a run:
    ``checkpoint.load_reference_checkpoint(path, g_running=G)``); it is put in eval mode.  renderer: a
    ``DecaConditionRenderer`` on the same device; its image size is the condition's (256 in the reference), and the
    generator's condition pyramid resizes it to each of its resolutions.  resolution: 2**k output images.  mesh_albedo: the
    constant albedo of the mesh picture (see MESH_ALBEDO)."""

    def __init__(self, generator, renderer, resolution=256, batch_size=32, eye_centering=True, graphs=True,
                 mesh_albedo=MESH_ALBEDO):
        step = int(round(math.log2(resolution))) - 2 if resolution > 0 else -1
        if step < 1 or 4 * 2 ** step != resolution:
            raise ValueError(f"resolution must be a power of two >= 8, got {resolution}")
        if not (generator.rendered_flame_ascondition and generator.normal_maps_as_cond):
            raise ValueError("FlameSampler needs a generator conditioned on the texture render and the normal map "
                             "(rendered_flame_ascondition=True, normal_maps_as_cond=True)")
        if batch_size < 1:
            raise ValueError(f"batch_size must be positive, got {batch_size}")
        self.generator, self.renderer = generator.eval(), renderer
        self.resolution, self.step, self.batch_size = resolution, step, int(batch_size)
        self.eye_centering, self.graphs = bool(eye_centering), bool(graphs)
        self.device = renderer.flame.faces_tensor.device
        self._mesh_albedo = torch.full((self.batch_size, 3, FLAMETex.SIZE, FLAMETex.SIZE), float(mesh_albedo), device=self.device)
        self._captured = {}

    @torch.no_grad()
    def _batch(self, rows, identity):
        """One batch of exactly ``batch_size`` rows -> (images, conditions, mesh, cam, centred rows), fresh tensors."""
        B, S = rows.shape[0], self.renderer.image_size
        rows = rows.clone()
        p = split_deca(rows)
        verts, _ = self.renderer.flame.decode_vertices(p["shape"].contiguous(), p["exp"].contiguous(), p["pose"].contiguous())
        if self.eye_centering:
            cam = eye_camera(verts)
            a, b = DECA_SLICES["cam"]
            rows[:, a:b] = cam
        else:
            cam = p["cam"].contiguous()
        cond_u8 = self.renderer.render_vertices_u8(verts, cam, self.renderer.flametex(p["tex"]), p["lit"])
        mesh_u8 = self.renderer.render_vertices_u8(verts, cam, self._mesh_albedo, p["lit"])
        cond = torch.empty(B, 6, S, S, device=rows.device)
        u8_to_unit(cond_u8[:B], cond[:, 0:3])
        u8_to_unit(cond_u8[B:], cond[:, 3:6])
        mesh = image_to_u8(u8_to_unit(mesh_u8[:B], torch.empty(B, 3, S, S, device=rows.device)))
        img = self.generator(cond, step=self.step, alpha=1, input_indices=identity)[0]
        return image_to_u8(img), cond_u8, mesh, cam, rows

    def _replay(self, rows, identity):
        """``_batch`` through a CUDA graph captured for this input layout (after one eager warm-up on these inputs)."""
        key = (rows.shape[1], identity.dtype, tuple(identity.shape[1:]))
        ent = self._captured.get(key)
        if ent is None:
            static_in = (rows.clone(), identity.clone())
            self._batch(*static_in)                       # warm-up: workspaces, kernel attributes, the generator's mean_w
            torch.cuda.synchronize(self.device)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_out = self._batch(*static_in)
            ent = self._captured[key] = (graph, static_in, static_out)
        graph, static_in, static_out = ent
        static_in[0].copy_(rows)
        static_in[1].copy_(identity)
        graph.replay()
        return static_out

    @torch.no_grad()
    def sample(self, rows, identity_indices):
        """rows (N, >=236) float32 DECA rows on the device [shape | exp | pose | cam | tex | lit | ...]; identity_indices
        (N,) integer indices into the generator's identity embedding, or float32 (N, 512) z fed to the mapping network as
        ``StyledGenerator.forward`` accepts.  Returns a dict of device tensors:
            images      uint8 (N, R, R, 3)        the generated faces
            conditions  uint8 (2N, S, S, 3)       texture renders (0..N-1) and normal maps (N..2N-1), as ``render_u8``
            mesh        uint8 (N, S, S, 3)        the constant-albedo render, as the scripts save it
            cam         float32 (N, 3)            the camera used (eye-centred unless ``eye_centering=False``)
            rows        float32 (N, C)            a copy of ``rows`` with that camera in columns 156:159
        ``rows`` itself is not modified."""
        if rows.dim() != 2 or rows.shape[1] < DECA_COLUMNS or rows.dtype != torch.float32 or rows.device != self.device:
            raise ValueError(f"rows must be float32 (N, >={DECA_COLUMNS}) on {self.device}, got {rows.dtype} "
                             f"{tuple(rows.shape)} on {rows.device}")
        N = rows.shape[0]
        ident = identity_indices
        if ident.device != self.device or ident.shape[0] != N:
            raise ValueError(f"identity_indices must hold {N} entries on {self.device}")
        if ident.dtype != torch.float32:
            if ident.is_floating_point() or ident.dim() != 1:
                raise ValueError("identity_indices: (N,) integer indices or float32 (N, 512) z")
            ident = ident.long()
        B, S, R = self.batch_size, self.renderer.image_size, self.resolution
        out = {"images": torch.empty(N, R, R, 3, dtype=torch.uint8, device=self.device),
               "conditions": torch.empty(2 * N, S, S, 3, dtype=torch.uint8, device=self.device),
               "mesh": torch.empty(N, S, S, 3, dtype=torch.uint8, device=self.device),
               "cam": torch.empty(N, 3, device=self.device),
               "rows": torch.empty(N, rows.shape[1], device=self.device)}
        for b0 in range(0, N, B):
            n = min(B, N - b0)
            r, z = rows[b0:b0 + n], ident[b0:b0 + n]
            if n < B:                                     # pad with copies of the last row (samples do not interact)
                r = torch.cat([r, r[-1:].expand(B - n, *r.shape[1:])])
                z = torch.cat([z, z[-1:].expand(B - n, *z.shape[1:])])
            images, cond, mesh, cam, centred = self._replay(r, z) if self.graphs else self._batch(r.contiguous(), z.contiguous())
            out["images"][b0:b0 + n] = images[:n]
            out["conditions"][b0:b0 + n] = cond[:n]
            out["conditions"][N + b0:N + b0 + n] = cond[B:B + n]
            out["mesh"][b0:b0 + n] = mesh[:n]
            out["cam"][b0:b0 + n] = cam[:n]
            out["rows"][b0:b0 + n] = centred[:n]
        return out
