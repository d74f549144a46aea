#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY (build container) -- golden for FLAMETex (models/FLAME.py:220-242).

Runs the reference's UNMODIFIED ``FLAMETex`` on the CPU over the analytic texture space of
``gif_b200.flame_synth.synthetic_texture_space`` (side 512, n 50).  The reference reads ``tex_dir`` as (side*side*3, 200)
from an npz, so the space is written to a temporary npz with columns 50..199 zero (the reference keeps the first
``tex_params``); nothing of it is stored.  A seeded sample of output texels goes to tests/golden/flametex.npz, consumed by
tests/test_deca_conditions_gpu.py, which rebuilds the space analytically.   usage: python oracle/make_flametex_golden.py"""
import importlib
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from gif_b200.flame_synth import synthetic_texture_space  # noqa: E402

SIDE, N, B, SAMPLES = 512, 50, 4, 24576


def main():
    ref_import.load()
    ref_flame = importlib.import_module("my_utils.photometric_optimization.models.FLAME")
    mean, tex_dir = synthetic_texture_space(SIDE, N)
    full = np.zeros((tex_dir.shape[0], 200), np.float32)
    full[:, :N] = tex_dir
    texcode = torch.from_numpy((np.random.default_rng(5).standard_normal((B, N)) * 1.5).astype(np.float32))
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "tex_space.npz")
        np.savez_compressed(path, mean=mean, tex_dir=full)
        del full
        ftex = ref_flame.FLAMETex(types.SimpleNamespace(tex_space_path=path, tex_params=N))
    with torch.no_grad():
        albedo = ftex(texcode).numpy()                                           # (B,3,256,256) BGR
    rng = np.random.default_rng(6)
    idx = np.stack([rng.integers(0, s, SAMPLES) for s in albedo.shape], 1).astype(np.int16)
    vals = albedo[tuple(idx.T.astype(np.int64))]
    out = os.path.join(ROOT, "tests", "golden", "flametex.npz")
    np.savez_compressed(out, side=SIDE, n=N, texcode=texcode.numpy(), index=idx, albedo=vals.astype(np.float32),
                        albedo_abs_max=np.float32(np.abs(albedo).max()))
    print(f"flametex golden: {SAMPLES} texels of ({B},3,256,256), |albedo| max {np.abs(albedo).max():.1f} -> {out}")


if __name__ == "__main__":
    main()
