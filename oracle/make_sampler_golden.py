#!/usr/bin/env python
"""Container-only: runs the *unmodified* reference ``position_to_given_location`` (my_utils/eye_centering.py:35-66) on the
CPU over 64 seeded DECA rows, decoded by the FLAME oracle (oracle/flame_oracle.py) on the synthetic FLAME-shaped model --
which has the real topology (V = 5023), so the eye vertices 4051 / 4597 exist -- and writes tests/golden/eye_centering.npz:
the rows, the two float32 eye vertices of every row (all the function reads of the mesh), the cam columns it wrote, and the
float64 vertices' eyes.  The distance of the float64 restatement (oracle/eye_centering_oracle.py) from the reference's
float32 pseudo-inverse goes to tests/golden/EYE_CENTERING_ORACLE_VS_REFERENCE.txt; the tests use it as their bar.
usage: python oracle/make_sampler_golden.py"""
import contextlib
import importlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import eye_centering_oracle as EO  # noqa: E402
from oracle import flame_oracle as FO  # noqa: E402
from oracle import ref_import  # noqa: E402
from gif_b200.flame_synth import synthetic_deca_params, synthetic_flame_model  # noqa: E402

N, SEED = 64, 31


def main():
    ref_import.load()
    with contextlib.redirect_stdout(io.StringIO()):
        ref_eye = importlib.import_module("my_utils.eye_centering")
    m = synthetic_flame_model()
    rows = synthetic_deca_params(N, SEED)
    decoded = {}

    def decoder(shape_params, expression_params, pose_params):      # the reference calls deca_flame_decoder(**params)
        out = FO.flame_forward(m, shape_params, expression_params, pose_params)
        decoded["verts"] = out[0]
        return out

    ref_rows = ref_eye.position_to_given_location(decoder, rows.clone())
    verts32 = decoded["verts"]
    i1, i2 = EO.EYE_VERTICES
    eyes32 = torch.stack([verts32[:, i1], verts32[:, i2]], 1).numpy()
    cam_ref = ref_rows[:, 156:159].numpy()
    assert torch.equal(ref_rows[:, :156], rows[:, :156]) and torch.equal(ref_rows[:, 159:], rows[:, 159:])
    verts64 = FO.flame_forward(m, rows[:, :100].double(), rows[:, 100:150].double(), rows[:, 150:156].double())[0]
    eyes64 = torch.stack([verts64[:, i1], verts64[:, i2]], 1).numpy()

    cam64 = EO.eye_camera(eyes32[:, 0], eyes32[:, 1])
    pinv_err = np.abs(cam64 - cam_ref.astype(np.float64)).max(0)                 # per column: s, bx, by
    vert_err = np.abs(EO.eye_camera(eyes64[:, 0], eyes64[:, 1]) - cam64).max(0)  # what float32 decoding alone moves
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "eye_centering.npz"), rows=rows.numpy(), eyes=eyes32,
                        eyes_f64=eyes64, cam_ref=cam_ref, pinv_err=pinv_err, vert_err=vert_err,
                        eye_vertices=np.int64(EO.EYE_VERTICES), targets=EO.EYE_TARGETS.astype(np.float32))
    cols = ("scale", "tx", "ty")
    lines = [f"# oracle/eye_centering_oracle.py (float64 closed form) vs the unmodified reference position_to_given_location "
             f"(float32 torch.pinverse), {N} rows, synthetic FLAME-shaped model, written by oracle/make_sampler_golden.py",
             f"# cam magnitude: |scale| {np.abs(cam_ref[:, 0]).min():.3f}..{np.abs(cam_ref[:, 0]).max():.3f}, "
             f"|tx|,|ty| <= {np.abs(cam_ref[:, 1:]).max():.3e}"]
    lines += [f"cam[{c}] max|oracle(f32 verts) - reference| = {e:.3e}" for c, e in zip(cols, pinv_err)]
    lines += [f"cam[{c}] max|oracle(f64 verts) - oracle(f32 verts)| = {e:.3e}" for c, e in zip(cols, vert_err)]
    with open(os.path.join(ROOT, "tests", "golden", "EYE_CENTERING_ORACLE_VS_REFERENCE.txt"), "w") as fh:
        fh.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
