"""GPU: the large CTA tiles of the wgmma implicit-GEMM convolution (128 sites x 256 channels when Co % 256 == 0, else
256 sites x 128 channels; one CTA per SM) against the exact-fp32 SIMT kernel, in tf32 (pre-rounded inputs, bar 2e-5) and
bf16x3 (raw inputs, bar 5e-5), and which tile the host picks for a shape."""
import math

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import golden_util as gu

pytestmark = pytest.mark.gpu


def run(x, w, k, mode, flip, transposed, impl):
    from gif_b200 import ops
    old = ops.CONV_IMPL
    ops.CONV_IMPL = impl
    try:
        y, _ = ops._conv_raw(x, w, k, mode, flip, transposed,
                             (ops.conv_out_size(x.shape[1], k, mode), ops.conv_out_size(x.shape[2], k, mode)))
    finally:
        ops.CONV_IMPL = old
    return y


def inputs(B, Hs, Ws, Ci, Co, k, mode, transposed, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    Hi, Wi = (Hs, Ws) if mode != 1 else (2 * Hs + 1, 2 * Ws + 1)
    x = torch.randn(B, Hi, Wi, Ci, device=dev, generator=g)
    wshape = (k * k, Ci, Co) if transposed else (k * k, Co, Ci)
    w = torch.randn(*wshape, device=dev, generator=g) / math.sqrt(Ci * k * k)
    return x, w


# (B, Hs, Ws, Ci, Co, k, mode)   Hs/Ws = SITE grid (output for S1/S2, input for T2).  Every case has at least 132 large
# tiles, so it runs on them: boxes of one row, of two rows (W = 256 / 128), and of several whole images with a batch that
# is not a multiple of the images per box (8x8: 4 per 256-site box; 4x4: 8 per 128-site box).
CASES = [
    (3, 64, 128, 32, 256, 3, 0), (1, 256, 256, 32, 128, 3, 0), (526, 8, 8, 32, 128, 3, 0),
    (3, 64, 64, 32, 512, 3, 1), (3, 128, 128, 32, 128, 3, 1), (523, 4, 4, 32, 512, 3, 1),
    (17, 16, 16, 32, 256, 3, 2), (130, 8, 8, 64, 128, 3, 2),
]


@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", CASES)
@pytest.mark.parametrize("flip,transposed", [(False, False), (True, True), (False, True)])
def test_large_tile_tf32_matches_simt(cuda, B, Hs, Ws, Ci, Co, k, mode, flip, transposed):
    from gif_b200 import ops
    x, w = inputs(B, Hs, Ws, Ci, Co, k, mode, transposed, B * 1000 + Hs + Ci + mode, cuda)
    x, w = ops._round_tf32_raw(x), ops._round_tf32_raw(w)
    y_tc = run(x, w, k, mode, flip, transposed, 2)
    y_ref = run(x, w, k, mode, flip, transposed, 1)
    torch.cuda.synchronize()
    assert y_tc.shape == y_ref.shape
    e = gu.rel_err(y_tc.cpu().numpy(), y_ref.cpu().numpy())
    assert e < 2e-5, e


@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", CASES)
@pytest.mark.parametrize("flip,transposed", [(False, False), (True, True), (False, True)])
def test_large_tile_bf16x3_matches_exact_fp32(cuda, B, Hs, Ws, Ci, Co, k, mode, flip, transposed):
    x, w = inputs(B, Hs, Ws, Ci, Co, k, mode, transposed, B * 1000 + Hs + Ci + mode + 5, cuda)
    y_x3 = run(x, w, k, mode, flip, transposed, 3)
    y_ref = run(x, w, k, mode, flip, transposed, 1)
    torch.cuda.synchronize()
    e = gu.rel_err(y_x3.cpu().numpy(), y_ref.cpu().numpy())
    assert 1e-8 < e < 5e-5, e        # > 1e-8: not the SIMT kernel again


def conv_kernel_names(fn):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages() if "conv_tc_kernel" in e.key}


@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode,tile", [
    (3, 64, 128, 32, 256, 3, 0, "<128, 256, true>"),     # Co % 256 == 0, 192 large tiles
    (1, 256, 256, 32, 128, 3, 0, "<256, 128, true>"),    # Co == 128, 256 large tiles
    (16, 16, 16, 64, 512, 3, 0, "<128, 128, true>"),     # 64 large tiles: too few for one CTA per SM
    (32, 4, 4, 512, 512, 3, 0, "<128, 128, true>"),      # split-K schedule
    (2, 16, 16, 32, 32, 3, 0, "<128, 32, true>"),        # Co < 128
])
def test_tile_choice(cuda, B, Hs, Ws, Ci, Co, k, mode, tile):
    x, w = inputs(B, Hs, Ws, Ci, Co, k, mode, False, 3, cuda)
    run(x, w, k, mode, False, False, 3)          # load the module and stage the weights outside the profiled call
    names = conv_kernel_names(lambda: run(x, w, k, mode, False, False, 3))
    assert len(names) == 1 and tile in next(iter(names)), names
