"""Training conditions rendered on the device from DECA parameters (SURVEY 8f.1): the 6-channel condition of the flagship
configuration (texture render + normal map) made from a dataset row instead of read from the render LMDB that
prepare_lmdb/create_deca_rendered_lmdb.py writes.

That script hands each row's [shape | exp | pose | cam | tex | lit] to ``OverLayViz.get_rendered_mesh``
(visualize_flame_overlay.py:17-33: gif_helper.render_tex_and_normal, then floor / clamp quantisation) and stores
``(x * 255).astype('uint8')`` of both images as PNG.  ``floor(clamp(t, 0, 255)) / 255 * 255`` cast to uint8 is exactly
``floor(clamp(t, 0, 255))`` in float32 (likewise for the normal map), and PNG is lossless, so ``render_u8`` returns the bytes
the LMDB holds, in the layout the device PNG decoder writes; ``__call__`` then maps them to [-1, 1] as the loader does.

Parity: the bytes match the reference's LMDB as far as the pytorch3d-convention rasteriser matches pytorch3d, which is
unpinned (gif_b200.render); against the reference's own Renderer on the rasterisation oracle the quantised maps differ by at
most one level on isolated pixels (tests/test_render_gpu.py)."""
import torch

from .image_decode import u8_to_unit
from .render import FlameRenderer, batch_orth_proj

# column ranges of a DECA parameter row (the reference's constants.INDICES / DECA_IDX)
DECA_SLICES = {"shape": (0, 100), "exp": (100, 150), "pose": (150, 156), "cam": (156, 159), "tex": (159, 209),
               "lit": (209, 236)}
DECA_COLUMNS = 236


def split_deca(deca):
    """(B, >=236) rows -> dict of column views: shape (B,100), exp (B,50), pose (B,6), cam (B,3), tex (B,50),
    lit (B,9,3)."""
    if deca.dim() != 2 or deca.shape[1] < DECA_COLUMNS:
        raise ValueError(f"DECA parameter rows need at least {DECA_COLUMNS} columns "
                         f"[shape 100 | exp 50 | pose 6 | cam 3 | tex 50 | lit 27], got {deca.shape[-1] if deca.dim() else 0} "
                         f"(shape {tuple(deca.shape)})")
    out = {k: deca[:, a:b] for k, (a, b) in DECA_SLICES.items()}
    out["lit"] = out["lit"].reshape(-1, 9, 3)
    return out


class DecaConditionRenderer:
    """Renders the (texture, normal map) condition of DECA rows on the device: FLAME decoder -> FLAMETex -> weak-perspective
    camera -> rasteriser + shading, ``image_size`` = the dataset's ``rend_flm_res``.  Build it from a
    ``gif_b200.flame.FLAME``, a ``gif_b200.flame.FLAMETex`` (both on the device) and the template's UVs."""

    def __init__(self, flame, flametex, uvcoords, uvfaces, image_size=256, convention="pytorch3d"):
        self.flame, self.flametex, self.image_size = flame, flametex, image_size
        dev = flame.faces_tensor.device
        self.renderer = FlameRenderer(flame.faces_tensor.cpu(), uvcoords, uvfaces, image_size, convention).to(dev)

    @torch.no_grad()
    def render_u8(self, deca, out=None):
        """deca (B, >=236) float32 CUDA, RAW parameter rows (not normalised labels) -> uint8 (2B, S, S, 3): planes 0..B-1
        the textured renders, planes B..2B-1 the normal maps.  ``out``: an optional tensor of that shape to write into."""
        p = split_deca(deca.float())
        verts, _ = self.flame.decode_vertices(p["shape"].contiguous(), p["exp"].contiguous(), p["pose"].contiguous())
        return self.render_vertices_u8(verts, p["cam"].contiguous(), self.flametex(p["tex"]), p["lit"], out)

    @torch.no_grad()
    def render_vertices_u8(self, verts, cam, albedo, lights, out=None):
        """The render of ``render_u8`` from decoded vertices (B,V,3), cameras (B,3), albedo (B,3,T,T) and lights (B,9,3):
        -> uint8 (2B, S, S, 3), textured renders then normal maps (into ``out`` when given)."""
        B, S = verts.shape[0], self.image_size
        trans = batch_orth_proj(verts, cam)                                          # gif_helper.py:25-27
        trans[:, :, 1:] = -trans[:, :, 1:]
        out = torch.empty(2 * B, S, S, 3, dtype=torch.uint8, device=verts.device) if out is None else out
        self.renderer(verts, trans, albedo, lights, want_cond=False, cond_u8=out)
        return out

    def __call__(self, deca):
        """deca (B, >=236) -> condition (B, 6, S, S) float32 in [-1, 1], what the loader yields for these rows."""
        u8 = self.render_u8(deca)
        B, S = deca.shape[0], self.image_size
        cond = torch.empty(B, 6, S, S, device=deca.device)
        u8_to_unit(u8[:B], cond[:, 0:3])
        u8_to_unit(u8[B:], cond[:, 3:6])
        return cond
