"""FLAME conditioning render on the GPU: (vertices, camera-projected vertices, albedo, SH lights) -> textured image,
normal image and the 6-channel condition map the generator consumes.

Follows the arithmetic of the reference's render path
    gif_helper.render_utils.render_tex_and_normal   (my_utils/photometric_optimization/gif_helper.py:24-40)
    Renderer.forward / add_SHlight / render_normal  (my_utils/photometric_optimization/renderer.py:130-221,291-305)
    util.vertex_normals / face_vertices / batch_orth_proj (my_utils/photometric_optimization/util.py:73-83,135-189)
    OverLayViz.get_rendered_mesh quantisation       (my_utils/visualize_flame_overlay.py:29-31)
Two rasterisation conventions (``FlameRenderer(..., convention=...)``), the choice stated, not hidden:
  "pytorch3d" (default) -- what the reference's conditioning maps are actually made with: pytorch3d ``rasterize_meshes`` as
               ``Pytorch3dRasterizer.forward`` calls it (renderer.py:46-67: NDC with x, y negated, pixel centres at +0.5,
               no back-face culling, linear depth, strictly-inside test), gifb200_rasterize_fwd_ex convention 1.  The fork the
               reference pins is absent and unversioned (SURVEY 8c): PARITY UNPINNED, checked against the restatement of
               the published rules in oracle/rasterize_oracle.c;
  "standard"  -- the in-repo ``standard_rasterize`` semantics (gif_b200.rasterize: pixel centres at integer coordinates
               after the visibility.py:38-40 mapping, front faces only, perspective-interpolated depth), bit-exact against
               the reference's own kernels.
Everything downstream of the (triangle, bary) buffers is the reference's formulae, fused into one kernel
(gifb200_render_shade).

Conditioning maps are *data* for the GAN (the reference detaches every attribute, renderer.py:149-150), so this path is
forward-only; the differentiable rasteriser itself is gif_b200.rasterize.rasterize.
"""
import torch

from . import rasterize
from ._lib import check, lib, ptr, require_cuda, stream


def batch_orth_proj(X, camera):
    """util.py:73-83: (s, tx, ty) weak-perspective camera."""
    camera = camera.reshape(-1, 1, 3)
    X_trans = torch.cat([X[:, :, :2] + camera[:, :, 1:], X[:, :, 2:]], 2)
    return camera[:, :, 0:1] * X_trans


def face_vertices(vertices, faces):
    """util.py:135-153: (B,V,C) gathered by (F,3) -> (B,F,3,C)."""
    return vertices[:, faces]


def vertex_adjacency(faces, V):
    """The vertex -> face-corner CSR adjacency ``gifb200_vertex_normals`` sums over, built once per topology: (faces (F,3)
    int32, offsets (V+1) int32, corners (3F) int32 = f*3 + corner, ascending within each vertex), on ``faces``' device."""
    flat = faces.reshape(-1).long()
    _, corners = torch.sort(flat, stable=True)
    offsets = torch.zeros(V + 1, dtype=torch.long, device=faces.device)
    offsets[1:] = torch.cumsum(torch.bincount(flat, minlength=V), 0)
    return faces.int().contiguous(), offsets.int(), corners.int()


def vertex_normals(vertices, faces, adjacency=None, face_normals=False):
    """util.py:156-189: area-weighted vertex normals, normalised (eps 1e-6), on ``gifb200_vertex_normals``: a fixed-order
    sum per vertex, bitwise reproducible.  ``adjacency``: ``vertex_adjacency(faces, V)``, built here when not given.
    -> normals (B,V,3), and with ``face_normals`` also the per-corner gather (B,F,3,3) from the same launch."""
    B, V = vertices.shape[:2]
    v = vertices.contiguous().float()
    require_cuda(v)
    fi, off, adj = vertex_adjacency(faces.to(v.device), V) if adjacency is None else adjacency
    F_ = fi.shape[0]
    if off.shape[0] != V + 1:
        raise ValueError(f"vertex_normals: the adjacency covers {off.shape[0] - 1} vertices, the mesh has {V}")
    n = torch.empty(B, V, 3, device=v.device)
    fn = torch.empty(B, F_, 3, 3, device=v.device) if face_normals else None
    check(lib.gifb200_vertex_normals(ptr(v), ptr(fi), ptr(off), ptr(adj), ptr(n), ptr(fn), B, V, F_, stream()),
          "gifb200_vertex_normals")
    return (n, fn) if face_normals else n


class FlameRenderer(torch.nn.Module):
    """Renderer (renderer.py:87-127) for a fixed topology: faces (F,3), per-corner UVs from (uvcoords (Vt,2), uvfaces (F,3))."""

    def __init__(self, faces, uvcoords, uvfaces, image_size=256, convention="pytorch3d"):
        super().__init__()
        if convention not in rasterize.CONVENTIONS:
            raise ValueError(f"convention must be one of {sorted(rasterize.CONVENTIONS)}")
        self.convention = convention
        self.image_size = image_size
        self.register_buffer("faces", faces.long())
        uv = torch.cat([uvcoords, torch.ones_like(uvcoords[:, :1])], -1) * 2 - 1       # renderer.py:107-109
        uv[:, 1] = -uv[:, 1]
        self.register_buffer("face_uv", uv[uvfaces.long()][:, :, :2].contiguous().float())   # (F,3,2) grid coordinates
        self._adjacency = None

    def adjacency(self, V):
        """``vertex_adjacency`` of this renderer's faces on their device, built on first use."""
        a = self._adjacency
        if a is None or a[1].shape[0] != V + 1 or a[0].device != self.faces.device:
            a = self._adjacency = vertex_adjacency(self.faces, V)
        return a

    @torch.no_grad()
    def forward(self, vertices, transformed_vertices, albedos, lights, want_cond=True, cond_u8=None):
        """vertices (B,V,3) world space; transformed_vertices (B,V,3) projected to [-1,1] (x right, y down after the flip
        of gif_helper.py:27); albedos (B,3,T,T); lights (B,9,3).  Returns dict(images (B,3,H,W), normal_images (B,3,H,W),
        alpha (B,1,H,W), cond (B,6,H,W) in [-1,1], triangle (B,H,W)).  ``cond_u8``: an optional uint8 (2B,H,W,3) tensor
        that receives the quantised texture (planes 0..B-1) and normal (planes B..2B-1) images as the reference's render
        LMDB stores them."""
        B = vertices.shape[0]
        H = W = self.image_size
        tv = transformed_vertices.clone().float()
        tv[:, :, 2] = tv[:, :, 2] + 10                                             # renderer.py:139
        pix = tv.clone()
        if self.convention == "pytorch3d":
            pix[..., :2] = -pix[..., :2]                                           # renderer.py:54-55, NDC in
            depth0 = float("inf")
        else:                                                                      # visibility.py:38-40 pixel mapping
            pix[..., 0] = tv[..., 0] * W / 2 + W / 2
            pix[..., 1] = tv[..., 1] * H / 2 + H / 2
            pix[..., 2] = tv[..., 2] - tv[..., 2].min() + 1
            depth0 = 1e6
        fv = face_vertices(pix, self.faces).contiguous()
        normals, fn = vertex_normals(vertices, self.faces, self.adjacency(vertices.shape[1]), face_normals=True)  # renderer.py:143
        depth = torch.full((B, H, W), depth0, device=fv.device)
        tri = torch.full((B, H, W), -1, dtype=torch.int32, device=fv.device)
        bary = torch.zeros((B, H, W, 3), device=fv.device)
        rasterize._forward(fv, None, depth, tri, bary, H, W, convention=self.convention)
        tex = torch.empty((B, H, W, 3), device=fv.device)
        nrm = torch.empty((B, H, W, 3), device=fv.device)
        cond = torch.empty((B, H, W, 6), device=fv.device) if want_cond else None
        alb = albedos.contiguous().float()
        sh = lights.contiguous().float()
        if cond_u8 is not None and (cond_u8.shape != (2 * B, H, W, 3) or cond_u8.dtype != torch.uint8 or
                                    not cond_u8.is_contiguous()):
            raise ValueError(f"cond_u8 must be a contiguous uint8 ({2 * B}, {H}, {W}, 3) tensor")
        check(lib.gifb200_render_shade(ptr(tri), ptr(bary), ptr(self.face_uv), ptr(fn), ptr(alb), ptr(sh), ptr(tex), ptr(nrm),
                                       ptr(cond), ptr(cond_u8), B, self.faces.shape[0], H, W, alb.shape[-1], stream()),
              "gifb200_render_shade")
        return {"images": tex.permute(0, 3, 1, 2), "normal_images": nrm.permute(0, 3, 1, 2),
                "alpha": (tri >= 0).float()[:, None], "cond": None if cond is None else cond.permute(0, 3, 1, 2),
                "triangle": tri, "normals": normals}

    def render_tex_and_normal(self, verts, cam, albedos, lights):
        """gif_helper.py:24-40 for given world vertices: orthographic projection, y/z flip, render."""
        trans = batch_orth_proj(verts, cam)
        trans[:, :, 1:] = -trans[:, :, 1:]
        out = self.forward(verts, trans, albedos, lights)
        return out["images"], out["normal_images"], out["cond"]
