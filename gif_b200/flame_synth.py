"""Synthetic FLAME-shaped workload for the rasteriser (BASELINE.json configs[3], SURVEY 8d config 4).

The FLAME model itself (generic_model.pkl, texture space) is licence-gated and absent from the reference tree, so
"random FLAME params" drive a FLAME-*shaped* linear decoder on the real FLAME topology (V=5023, F=9976; template from
my_utils/photometric_optimization/data/head_template_mesh.obj, stored as tests/golden/flame_template.npz):
    verts = T + sum_j beta_j S_j,  beta ~ N(0,1) (B,150)
with a SMOOTH basis S_j(v) = a * d_j * cos(2 pi f_j . T_v + phi_j) (|f_j| <= 8 cycles/m, a = 0.5 mm, i.e. ~4 mm rms total
displacement, comparable to FLAME's shape+expression range).  (SURVEY 8d suggested i.i.d. per-vertex noise N(0,(2 mm)^2)
per coefficient; that sums to 24 mm rms of *uncorrelated* vertex noise, which crumples the mesh into image-sized slivers
(mean bbox 1800 px^2 at 256^2) and no longer resembles a FLAME render, so it is not used.)  It is followed by the reference's camera path: a random head rotation (cf. plots/generate_random_samples.py:107-108),
util.batch_orth_proj (util.py:73-83) + the y/z flip of gif_helper.py:26-27, and the pixel mapping of
visibility.py:38-40 (x*w/2+w/2, y*h/2+h/2, z-min(z)+1).
"""
import math
import os

import numpy as np
import torch

_TEMPLATE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                         "flame_template.npz")
_cache = {}


def flame_topology():
    if "t" not in _cache:
        z = np.load(_TEMPLATE)
        v = torch.from_numpy(z["vertices"].astype(np.float32))
        _cache["t"] = (v - v.mean(0, keepdim=True), torch.from_numpy(z["faces"].astype(np.int64)))
    return _cache["t"]


def flame_uv():
    """(uvcoords (5118,2), uvfaces (9976,3)) of the FLAME template."""
    z = np.load(_TEMPLATE)
    return torch.from_numpy(z["uvcoords"].astype(np.float32)), torch.from_numpy(z["uvfaces"].astype(np.int64))


def synthetic_flame_params(batch, seed=0):
    """World-space vertices (B,V,3), weak-perspective cameras (B,3), albedo textures (B,3,256,256) in 0..255 and SH lights
    (B,9,3) for the render benchmark: the smooth FLAME-shaped decoder below + random pose / camera / smooth random albedo."""
    tmpl, faces = flame_topology()
    g = torch.Generator().manual_seed(4321 + seed)
    verts = _decode(batch, g, tmpl)
    cam = torch.cat([torch.rand(batch, 1, generator=g) * 3 + 7, (torch.rand(batch, 2, generator=g) * 2 - 1) * 0.02], 1)
    low = torch.rand(batch, 3, 8, 8, generator=g) * 255
    albedo = torch.nn.functional.interpolate(low, size=(256, 256), mode="bilinear", align_corners=False)
    lights = torch.zeros(batch, 9, 3)
    lights[:, 0] = 3.0 + 0.3 * torch.randn(batch, 3, generator=g)
    lights[:, 1:] = 0.3 * torch.randn(batch, 8, 3, generator=g)
    return verts, cam, albedo, lights


def _decode(batch, g, tmpl):
    gb = torch.Generator().manual_seed(7)
    freq = (torch.rand(150, 3, generator=gb) * 2 - 1) * 8.0
    phase = torch.rand(150, 1, generator=gb) * (2 * math.pi)
    dirs = torch.nn.functional.normalize(torch.randn(150, 3, generator=gb), dim=1)
    wave = torch.cos(2 * math.pi * (freq @ tmpl.t()) + phase)
    basis = (0.0005 * wave[:, :, None] * dirs[:, None, :]).reshape(150, -1)
    beta = torch.randn(batch, 150, generator=g)
    verts = tmpl[None] + (beta @ basis).reshape(batch, -1, 3)
    yaw = (torch.rand(batch, generator=g) * 2 - 1) * (math.pi / 8)
    pitch = torch.rand(batch, generator=g) * (math.pi / 12)
    cy, sy, cp, sp = torch.cos(yaw), torch.sin(yaw), torch.cos(pitch), torch.sin(pitch)
    zero, one = torch.zeros_like(cy), torch.ones_like(cy)
    ry = torch.stack([cy, zero, sy, zero, one, zero, -sy, zero, cy], -1).reshape(batch, 3, 3)
    rx = torch.stack([one, zero, zero, zero, cp, -sp, zero, sp, cp], -1).reshape(batch, 3, 3)
    return verts @ (rx @ ry).transpose(1, 2)


def synthetic_flame_batch(batch, h, w, seed=0, device="cuda"):
    """-> face_vertices (B,F,3,3) fp32 in pixel space, face_colors (B,F,3,3) in [0,1]."""
    tmpl, faces = flame_topology()
    g = torch.Generator().manual_seed(1234 + seed)
    verts = _decode(batch, g, tmpl)
    cam = torch.cat([torch.rand(batch, 1, generator=g) * 3 + 7, (torch.rand(batch, 2, generator=g) * 2 - 1) * 0.02], 1)
    proj = torch.cat([verts[..., :2] + cam[:, None, 1:], verts[..., 2:]], -1) * cam[:, None, 0:1]   # batch_orth_proj
    proj[..., 1:] = -proj[..., 1:]                                                                   # gif_helper.py:27
    pix = proj.clone()
    pix[..., 0] = proj[..., 0] * w / 2 + w / 2
    pix[..., 1] = proj[..., 1] * h / 2 + h / 2
    pix[..., 2] = proj[..., 2] - proj[..., 2].min() + 1
    vcol = torch.rand(batch, tmpl.shape[0], 3, generator=g)
    fv = pix[:, faces]          # (B,F,3,3)
    fc = vcol[:, faces]
    return fv.contiguous().to(device), fc.contiguous().to(device)


def synthetic_flame_model(seed=11, n_shape=100, n_exp=50):
    """A FLAME-*shaped* articulated model on the real FLAME topology (the licence-gated generic_model.pkl is absent): the
    tensors FLAME.__init__ registers (FLAME.py:50-68, 80-86) with the same shapes / meaning, filled deterministically:
      v_template (V,3); shapedirs (V,3,n_shape+n_exp): the smooth basis of ``_decode``; posedirs (36, V*3): smooth, ~0.3 mm
      per unit of pose feature; J_regressor (5,V): rows >= 0 summing to 1 (Gaussian windows around 5 joint centres: root,
      neck, jaw, two eyes); parents [-1,0,1,1,1] (FLAME's kinematic tree); lbs_weights (V,5): softmax of -dist^2 to the
      joint centres (rows sum to 1); landmark embeddings: 51 static, 79 x 17 dynamic, 68 full (random faces / barycentrics).
    Everything is float32 CPU tensors; pass to gif_b200.flame.FLAME.from_arrays."""
    tmpl, faces = flame_topology()
    V = tmpl.shape[0]
    g = torch.Generator().manual_seed(seed)
    nb = n_shape + n_exp
    freq = (torch.rand(nb, 3, generator=g) * 2 - 1) * 8.0
    phase = torch.rand(nb, 1, generator=g) * (2 * math.pi)
    dirs = torch.nn.functional.normalize(torch.randn(nb, 3, generator=g), dim=1)
    wave = torch.cos(2 * math.pi * (freq @ tmpl.t()) + phase)                         # (nb, V)
    shapedirs = (0.0005 * wave[:, :, None] * dirs[:, None, :]).permute(1, 2, 0).contiguous()   # (V,3,nb)
    freq = (torch.rand(36, 3, generator=g) * 2 - 1) * 6.0
    phase = torch.rand(36, 1, generator=g) * (2 * math.pi)
    dirs = torch.nn.functional.normalize(torch.randn(36, 3, generator=g), dim=1)
    wave = torch.cos(2 * math.pi * (freq @ tmpl.t()) + phase)
    posedirs = (0.0003 * wave[:, :, None] * dirs[:, None, :]).reshape(36, V * 3).contiguous()
    lo, hi = tmpl.min(0).values, tmpl.max(0).values
    ext = hi - lo
    centres = torch.stack([lo + ext * torch.tensor(f) for f in
                           ([0.5, 0.15, 0.35], [0.5, 0.3, 0.4], [0.5, 0.4, 0.75], [0.33, 0.62, 0.85], [0.67, 0.62, 0.85])])
    d2 = ((tmpl[None] - centres[:, None]) ** 2).sum(-1)                               # (5,V)
    jr = torch.exp(-d2 / (2 * (0.02 ** 2)))
    jr = jr / jr.sum(1, keepdim=True)
    lbs_weights = torch.softmax(-d2.t() / (2 * (0.03 ** 2)), dim=1).contiguous()     # (V,5)
    F_ = faces.shape[0]

    def bary(*shape):
        b = torch.rand(*shape, 3, generator=g) + 0.05
        return b / b.sum(-1, keepdim=True)

    return {
        "v_template": tmpl.clone(), "faces": faces.clone(), "shapedirs": shapedirs, "posedirs": posedirs,
        "J_regressor": jr.contiguous(), "parents": torch.tensor([-1, 0, 1, 1, 1], dtype=torch.long),
        "lbs_weights": lbs_weights, "n_shape": n_shape, "n_exp": n_exp,
        "lmk_faces_idx": torch.randint(0, F_, (51,), generator=g), "lmk_bary_coords": bary(51),
        "dynamic_lmk_faces_idx": torch.randint(0, F_, (79, 17), generator=g), "dynamic_lmk_bary_coords": bary(79, 17),
        "full_lmk_faces_idx": torch.randint(0, F_, (1, 68), generator=g), "full_lmk_bary_coords": bary(1, 68),
    }


def synthetic_texture_data(size=256):
    """The pre-computed FLAME texture-space table FlameTextureSpace consumes (model/stg2_generator.py:349-354; the
    reference loads it from the licence-gated ``flame_texture_space_dat_file``): for every texel of the size x size UV
    atlas covered by a UV triangle, the three mesh VERTEX ids of that triangle (``valid_pixel_3d_faces``) and the
    barycentric weights of the texel centre (``valid_pixel_b_coords``).  Built here by rasterising the template's real UV
    layout (tests/golden/flame_template.npz): u -> column, (1 - v) -> row, texel centres at integer + 0.5."""
    if ("tex", size) in _cache:
        return _cache[("tex", size)]
    _, faces = flame_topology()
    uv, uvf = flame_uv()
    faces, uv, uvf = faces.numpy(), uv.numpy().astype(np.float64), uvf.numpy()
    px = np.stack([uv[:, 0] * size, (1.0 - uv[:, 1]) * size], 1)          # texel space, (x, y)
    tri = px[uvf]                                                         # (F,3,2)
    owner = -np.ones((size, size), dtype=np.int64)
    bary = np.zeros((size, size, 3), dtype=np.float64)
    for f in range(tri.shape[0]):
        (x0, y0), (x1, y1), (x2, y2) = tri[f]
        den = (y1 - y2) * (x0 - x2) + (x2 - x1) * (y0 - y2)
        if abs(den) < 1e-12:
            continue
        xa, xb = max(int(np.floor(min(x0, x1, x2) - 0.5)), 0), min(int(np.ceil(max(x0, x1, x2) - 0.5)), size - 1)
        ya, yb = max(int(np.floor(min(y0, y1, y2) - 0.5)), 0), min(int(np.ceil(max(y0, y1, y2) - 0.5)), size - 1)
        if xa > xb or ya > yb:
            continue
        xs, ys = np.meshgrid(np.arange(xa, xb + 1) + 0.5, np.arange(ya, yb + 1) + 0.5)
        w0 = ((y1 - y2) * (xs - x2) + (x2 - x1) * (ys - y2)) / den
        w1 = ((y2 - y0) * (xs - x2) + (x0 - x2) * (ys - y2)) / den
        w2 = 1.0 - w0 - w1
        inside = (w0 >= 0) & (w1 >= 0) & (w2 >= 0)
        sub_o, sub_b = owner[ya:yb + 1, xa:xb + 1], bary[ya:yb + 1, xa:xb + 1]
        take = inside & (sub_o < 0)
        sub_o[take] = f
        sub_b[take] = np.stack([w0, w1, w2], -1)[take]
    ys, xs = np.meshgrid(np.arange(size), np.arange(size), indexing="ij")
    valid = np.nonzero(owner.reshape(-1) >= 0)[0]
    data = {"x_coords": xs.reshape(-1).astype(np.int64), "y_coords": ys.reshape(-1).astype(np.int64),
            "valid_pixel_ids": valid.astype(np.int64),
            "valid_pixel_3d_faces": faces[owner.reshape(-1)[valid]].astype(np.int64),
            "valid_pixel_b_coords": bary.reshape(-1, 3)[valid].astype(np.float32)}
    _cache[("tex", size)] = data
    return data


def synthetic_texture_space(side=512, n=50):
    """A FLAMETex-shaped texture space (the licence-gated FLAME_texture.npz is absent), defined analytically so that it can
    be rebuilt anywhere instead of stored: texel (x, y), channel c, k = (y*side + x)*3 + c, u = x/side, v = y/side,
        mean[k]     = 128 + 60 cos(2 pi (1.5 u + 0.5 v) + 0.9 c)
        tex_dir[k,j] = 12 / (1 + 0.1 j) * cos(2 pi ((1 + j mod 5) u + (1 + 3j mod 7) v) + 0.37 j + (1.3 + 0.11 j) c)
    evaluated in float64 and rounded to float32.  -> (mean (side*side*3,), tex_dir (side*side*3, n)) numpy float32."""
    k = np.arange(side * side * 3, dtype=np.int64)
    c = (k % 3).astype(np.float64)
    u = ((k // 3) % side).astype(np.float64) / side
    v = (k // (3 * side)).astype(np.float64) / side
    mean = (128.0 + 60.0 * np.cos(2 * np.pi * (1.5 * u + 0.5 * v) + 0.9 * c)).astype(np.float32)
    tex_dir = np.empty((k.size, n), np.float32)
    for j in range(n):
        arg = 2 * np.pi * ((1 + j % 5) * u + (1 + (3 * j) % 7) * v) + 0.37 * j + (1.3 + 0.11 * j) * c
        tex_dir[:, j] = 12.0 / (1.0 + 0.1 * j) * np.cos(arg)
    return mean, tex_dir


def synthetic_deca_params(n, seed=0, cols=236):
    """(n, cols) DECA parameter rows [shape 100 | exp 50 | pose 6 | cam 3 | tex 50 | lit 27 | extra] in realistic ranges for
    the synthetic model: cam scale 7-10, yaw within +-pi/8, lights as ``synthetic_flame_params``."""
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros(n, cols)
    p[:, 0:100] = torch.randn(n, 100, generator=g)
    p[:, 100:150] = torch.randn(n, 50, generator=g) * 0.5
    p[:, 150] = torch.rand(n, generator=g) * 0.2 - 0.1                          # pitch
    p[:, 151] = (torch.rand(n, generator=g) * 2 - 1) * (math.pi / 8)           # yaw
    p[:, 153] = torch.rand(n, generator=g) * 0.2                                # jaw
    p[:, 156] = torch.rand(n, generator=g) * 3 + 7
    p[:, 157:159] = (torch.rand(n, 2, generator=g) * 2 - 1) * 0.02
    p[:, 159:209] = torch.randn(n, 50, generator=g)
    lit = torch.zeros(n, 9, 3)
    lit[:, 0] = 3.0 + 0.3 * torch.randn(n, 3, generator=g)
    lit[:, 1:] = 0.3 * torch.randn(n, 8, 3, generator=g)
    p[:, 209:236] = lit.reshape(n, 27)
    if cols > 236:
        p[:, 236:] = torch.randn(n, cols - 236, generator=g)
    return p
