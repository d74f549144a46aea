"""Eye-centred camera on the device: ``position_to_given_location`` (my_utils/eye_centering.py:35-66), which every sampling
script of the reference runs before rendering.  It decodes FLAME and replaces each row's camera (columns 156:159) by the
weak-perspective camera that places the two eye vertices 4051 / 4597 at fixed image positions.

The reference solves a 3x4 pseudo-inverse in float32, one row at a time in a Python loop; ``gifb200_eye_camera`` evaluates
the closed form of the same least-squares solution in float64 for the whole batch in one launch (include/gifb200.h).  A
row whose two eye vertices coincide in x and y has no unique camera: it gets NaN, as the reference divides by zero there
too; nothing checks for it on the host, so the call never waits for the device."""
import numpy as np
import torch

from ._lib import check, lib, ptr, require_cuda, stream
from .conditions import DECA_SLICES

EYE_VERTICES = (4051, 4597)
# normalized_image_desired_positions_x1_x2_y1_y2 (eye_centering.py:52-53), rounded to float32 as its torch.tensor is
EYE_TARGETS = tuple(float(v) for v in np.float32([-0.2419, 0.2441, 0.0501 - 0.1, 0.0509 - 0.1]))


def eye_camera(verts, eye_vertices=EYE_VERTICES, targets=EYE_TARGETS, out=None):
    """verts (B,V,3) float32 CUDA -> cam (B,3) = (scale, tx, ty) putting ``verts[:, eye_vertices[k], :2]`` at
    (targets[k], targets[2 + k]) under ``render.batch_orth_proj``; ``targets`` = (x1, x2, y1, y2).  ``out``: an optional
    contiguous float32 (B,3) tensor to write into."""
    v = verts.contiguous()
    require_cuda(v)
    if v.dim() != 3 or v.shape[2] != 3 or v.dtype != torch.float32:
        raise ValueError(f"eye_camera: verts must be float32 (B, V, 3), got {v.dtype} {tuple(v.shape)}")
    B, V = v.shape[:2]
    i1, i2 = (int(i) for i in eye_vertices)
    if not (0 <= i1 < V and 0 <= i2 < V):
        raise ValueError(f"eye_camera: eye vertices {i1}, {i2} outside the mesh's {V} vertices")
    if out is None:
        out = torch.empty(B, 3, device=v.device)
    elif out.shape != (B, 3) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError(f"eye_camera: out must be a contiguous float32 ({B}, 3) tensor")
    x1, x2, y1, y2 = (float(t) for t in targets)
    check(lib.gifb200_eye_camera(ptr(v), ptr(out), B, V, i1, i2, x1, x2, y1, y2, stream()), "gifb200_eye_camera")
    return out


def position_to_given_location(deca_flame_decoder, flame_batch):
    """eye_centering.py:35-66 with the reference's name and signature: decodes ``flame_batch`` (B, >=156) [shape | exp |
    pose | cam ...] with ``deca_flame_decoder`` (a ``gif_b200.flame.FLAME``), writes the eye-centred camera into columns
    156:159 IN PLACE and returns ``flame_batch``."""
    a, b = DECA_SLICES["cam"]
    if flame_batch.dim() != 2 or flame_batch.shape[1] < b:
        raise ValueError(f"position_to_given_location: rows need at least {b} columns, got shape {tuple(flame_batch.shape)}")
    col = lambda k: flame_batch[:, DECA_SLICES[k][0]:DECA_SLICES[k][1]].float().contiguous()
    verts, _ = deca_flame_decoder.decode_vertices(col("shape"), col("exp"), col("pose"))
    flame_batch[:, a:b] = eye_camera(verts)
    return flame_batch
