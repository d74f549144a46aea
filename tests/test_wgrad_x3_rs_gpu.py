"""GPU: the bf16x3 weight gradient as it runs by default -- S operand in registers, and for stride-1 3x3 layers one halo
tile of the big tensor shared by the three kw taps -- against the same kernel with both operands from shared memory and
one big-tensor tile per tap (GIFB200_WGRAD_X3_RS=0 GIFB200_WGRAD_HALO=0).  Both issue the same MMAs on the same values in
the same order into the same fp32 accumulators, so gw must be bitwise equal for every shape class of the X3 kernel.

The switches are read once per process, so each path runs in a child process (this file run as a script) that writes its
results to an .npz; the test compares the two files."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

CASES = [
    # (B, Hs, Ws, Ci, Co, k, mode)   Hs/Ws = SITE grid (output for S1/S2, input for T2)
    (3, 32, 32, 64, 128, 3, 0),       # S1 3x3 (halo tile), BLOCK_N 64, odd stage count per split
    (4, 128, 128, 128, 128, 3, 0),    # the 128 -> 128 3x3 layers of the 256^2 step (batch 4)
    (2, 16, 16, 32, 256, 3, 0),       # S1 3x3, BLOCK_N 32, two 128-row tiles
    (2, 16, 16, 64, 256, 1, 0),       # S1 1x1
    (2, 16, 16, 96, 128, 1, 0),       # S1 1x1, BLOCK_N 32
    (4, 4, 4, 64, 128, 3, 0),         # narrow images: one TMA box spans the rows (and images) of a stage
    (8, 8, 8, 32, 128, 3, 0),
    (1, 64, 64, 64, 128, 3, 1),       # S2
    (4, 4, 4, 64, 128, 3, 1),
    (1, 64, 64, 128, 128, 3, 2),      # T2
    (4, 4, 4, 128, 64, 3, 2),
    (2, 16, 16, 32, 32, 3, 0),        # STACK (Cs = 32), BLOCK_N 32
    (1, 64, 128, 64, 32, 3, 0),       # STACK, BLOCK_N 64
    (4, 4, 4, 32, 32, 3, 0),          # STACK, narrow images
    (1, 64, 64, 64, 64, 3, 0),        # narrow (AC = 2), Cs = 64
    (3, 8, 8, 64, 64, 3, 0),          # narrow, narrow images
    (3, 16, 16, 64, 64, 1, 0),        # narrow 1x1
    (2, 16, 32, 128, 64, 3, 1),       # narrow S2
    (1, 64, 64, 64, 32, 3, 2),        # narrow T2
    (3, 16, 16, 32, 64, 1, 0),        # narrow, Cs = 32 1x1 (the second chunk repeats the first)
    (2, 8, 8, 32, 32, 1, 0),
]
FLIPS = [(False, False), (True, True)]


def grids(Hs, Ws, mode):
    if mode == 0:
        return Hs, Ws, Hs, Ws
    if mode == 1:
        return 2 * Hs + 1, 2 * Ws + 1, Hs, Ws
    return Hs, Ws, 2 * Hs + 1, 2 * Ws + 1


def key(case, flip, transposed):
    return "_".join(str(v) for v in case) + f"_f{int(flip)}_t{int(transposed)}"


def compute(out):
    """Child: gw of every case on seeded inputs through the bf16x3 tensor-core weight gradient, into out (.npz)."""
    import torch
    from gif_b200 import ops
    from gif_b200._lib import lib
    dev = torch.device("cuda:0")
    ops.set_precision("bf16x3")
    res = {}
    for case in CASES:
        B, Hs, Ws, Ci, Co, k, mode = case
        Hi, Wi, Ho, Wo = grids(Hs, Ws, mode)
        assert lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, 3) == 3, case
        g = torch.Generator(device="cuda").manual_seed(B * 77 + Hs + Ci + Co + mode + k)
        x = torch.randn(B, Hi, Wi, Ci, device=dev, generator=g)
        gy = torch.randn(B, Ho, Wo, Co, device=dev, generator=g)
        for flip, transposed in FLIPS:
            res[key(case, flip, transposed)] = ops._wgrad_raw(x, gy, k, mode, flip, transposed).cpu().numpy()
    np.savez(out, **res)


@pytest.fixture(scope="module")
def both_paths(cuda, tmp_path_factory):
    d = tmp_path_factory.mktemp("wgrad_x3_rs")
    out = {}
    for rs in ("0", "1"):
        path = str(d / f"rs{rs}.npz")
        # "0": both operands from shared memory and one B tile per tap; "1": the defaults
        env = dict(os.environ, GIFB200_WGRAD_X3_RS=rs, GIFB200_WGRAD_HALO=rs)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), path], env=env, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        out[rs] = np.load(path)
    return out


@pytest.mark.parametrize("case", CASES, ids=lambda c: "_".join(str(v) for v in c))
@pytest.mark.parametrize("flip,transposed", FLIPS)
def test_wgrad_x3_registers_equal_shared_memory_bitwise(both_paths, case, flip, transposed):
    k = key(case, flip, transposed)
    ss, rs = both_paths["0"][k], both_paths["1"][k]
    assert ss.shape == rs.shape
    assert np.isfinite(rs).all() and np.abs(rs).max() > 0
    assert np.array_equal(ss.view(np.uint32), rs.view(np.uint32)), float(np.abs(ss - rs).max())


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    compute(sys.argv[1])
