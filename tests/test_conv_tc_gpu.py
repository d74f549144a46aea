"""GPU: the wgmma (tf32) implicit-GEMM convolution against the exact-fp32 SIMT kernel through the C ABI
(impl=2 vs impl=1), every mode / flag combination, tile-edge shapes (4x4 images packed 8 per tile, batch not a multiple of
the images-per-tile, ...).  Inputs are pre-rounded to tf32 so the only difference is the accumulation order: the bar is 2e-5
for those, and 1e-3 (BASELINE.json) for raw fp32 inputs through gif_b200.ops (which rounds)."""
import math

import pytest
import torch

import golden_util as gu

pytestmark = pytest.mark.gpu


def round_tf32(t):
    from gif_b200 import ops
    return ops._round_tf32_raw(t.contiguous())


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


CASES = [
    # (B, Hs, Ws, Ci, Co, k, mode)   Hs/Ws = SITE grid (output for S1/S2, input for T2)
    (2, 16, 16, 32, 32, 3, 0), (3, 4, 4, 64, 32, 3, 0), (5, 8, 8, 32, 64, 3, 0), (1, 32, 64, 64, 128, 3, 0),
    (2, 128, 128, 32, 128, 3, 0), (2, 16, 16, 96, 256, 1, 0), (1, 256, 256, 32, 32, 3, 0),
    (2, 16, 16, 32, 32, 3, 1), (3, 4, 4, 64, 64, 3, 1), (1, 64, 64, 32, 128, 3, 1), (2, 8, 32, 32, 32, 3, 1),
    (2, 16, 16, 32, 32, 3, 2), (3, 4, 4, 64, 64, 3, 2), (1, 64, 64, 32, 128, 3, 2), (2, 8, 32, 32, 32, 3, 2),
    # the small layers of the batch-32 step: 16 / 64 output tiles, run with the split-K schedule (16 / 4 splits)
    (32, 4, 4, 512, 512, 3, 0), (32, 4, 4, 512, 512, 3, 1), (32, 8, 8, 512, 512, 3, 1),
]


@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", CASES)
@pytest.mark.parametrize("flip,transposed", [(False, False), (True, True), (False, True)])
def test_tc_matches_simt(cuda, B, Hs, Ws, Ci, Co, k, mode, flip, transposed):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Hs + Ci + mode)
    Hi, Wi = (Hs, Ws) if mode != 1 else (2 * Hs + 1, 2 * Ws + 1)
    x = round_tf32(torch.randn(B, Hi, Wi, Ci, device=cuda, generator=g))
    wshape = (k * k, Ci, Co) if transposed else (k * k, Co, Ci)
    w = round_tf32(torch.randn(*wshape, device=cuda, generator=g) / math.sqrt(Ci * k * k))
    y_tc = run(x, w, k, mode, flip, transposed, 2)
    y_ref = run(x, w, k, mode, flip, transposed, 1)
    torch.cuda.synchronize()
    assert y_tc.shape == y_ref.shape
    e = gu.rel_err(y_tc.cpu().numpy(), y_ref.cpu().numpy())
    assert e < 2e-5, e


def test_tc_unrounded_inputs_within_1e3(cuda, tf32_mode):
    """fp32 inputs through the public op: the wrapper rounds to tf32 (round-to-nearest); result within 1e-3 of exact fp32."""
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(2, 64, 64, 128, device=cuda, generator=g)
    w = torch.randn(9, 128, 128, device=cuda, generator=g) / math.sqrt(1152)
    y = ops.conv2d(x, w, 3, ops.S1)
    ops.set_precision("fp32")
    y32 = ops.conv2d(x, w, 3, ops.S1)
    e = gu.rel_err(y.cpu().numpy(), y32.cpu().numpy())
    assert 1e-6 < e < 1e-3, e     # > 1e-6: the tensor-core path really ran


def test_tc_rejects_unsupported_shape(cuda):
    from gif_b200 import ops
    from gif_b200._lib import GifB200Error
    with pytest.raises(GifB200Error):
        run(torch.zeros(1, 9, 9, 32, device=cuda), torch.zeros(9, 32, 32, device=cuda), 3, 0, False, False, 2)


WG_CASES = [
    # (B, Hs, Ws, Ci, Co, k, mode)  site grid as above
    (2, 16, 16, 32, 128, 3, 0), (4, 4, 4, 64, 128, 3, 0), (1, 32, 64, 128, 128, 3, 0), (2, 64, 64, 32, 256, 3, 0),
    (2, 16, 16, 96, 128, 1, 0), (8, 8, 8, 32, 128, 3, 0),
    (2, 16, 16, 32, 128, 3, 1), (4, 4, 4, 64, 128, 3, 1), (1, 64, 64, 64, 128, 3, 1),
    (2, 16, 16, 128, 32, 3, 2), (4, 4, 4, 128, 64, 3, 2), (1, 64, 64, 128, 128, 3, 2),
    # STACK variant (Cs == 32): the zero-padded NoiseInjection convs
    (2, 16, 16, 32, 32, 3, 0), (4, 4, 4, 32, 32, 3, 0), (1, 64, 128, 64, 32, 3, 0), (3, 8, 8, 128, 32, 3, 0),
]


@pytest.mark.parametrize("impl", [2, 3])
@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", [(3, 4, 4, 64, 32, 3, 0), (32, 4, 4, 512, 512, 3, 1), (5, 8, 8, 32, 64, 3, 0)])
def test_splitk_with_fused_epilogue(cuda, B, Hs, Ws, Ci, Co, k, mode, impl):
    """Split-K layers with the fused bias + leaky-ReLU epilogue: the reduction pass applies it to the summed accumulator
    (tf32 and bf16x3 kernels vs the exact fp32 SIMT path with the same epilogue)."""
    from gif_b200 import ops
    from gif_b200._lib import lib
    g = torch.Generator(device="cuda").manual_seed(B + Hs + Ci + mode + 11)
    Hi, Wi = (Hs, Ws) if mode != 1 else (2 * Hs + 1, 2 * Ws + 1)
    ws_plain = k * k * Co * Ci * 4 + 512
    assert lib.gifb200_conv2d_workspace_bytes(B, Hi, Wi, Ci, Hs, Ws, Co, k, mode, 0, impl) > ws_plain, "shape is not on the split-K schedule"
    x = round_tf32(torch.randn(B, Hi, Wi, Ci, device=cuda, generator=g))
    w = round_tf32(torch.randn(k * k, Co, Ci, device=cuda, generator=g) / math.sqrt(Ci * k * k))
    bias = torch.randn(Co, device=cuda, generator=g)
    old = ops.CONV_IMPL
    try:
        outs = []
        for im in (impl, 1):
            ops.CONV_IMPL = im
            y, _ = ops._conv_raw(x, w, k, mode, False, False, (Hs, Ws), (bias, 0.2, math.sqrt(2.0), 0))
            outs.append(y)
    finally:
        ops.CONV_IMPL = old
    torch.cuda.synchronize()
    e = gu.rel_err(outs[0].cpu().numpy(), outs[1].cpu().numpy())
    assert e < (2e-5 if impl == 2 else 5e-5), e
    # deterministic: the partial sums are added in split order
    ops.CONV_IMPL = impl
    try:
        y2, _ = ops._conv_raw(x, w, k, mode, False, False, (Hs, Ws), (bias, 0.2, math.sqrt(2.0), 0))
    finally:
        ops.CONV_IMPL = old
    assert torch.equal(y2, outs[0])


@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", WG_CASES)
@pytest.mark.parametrize("flip,transposed", [(False, False), (True, True), (False, True)])
def test_wgrad_tc_matches_simt(cuda, B, Hs, Ws, Ci, Co, k, mode, flip, transposed):
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 77 + Hs + Ci + mode)
    if mode == 0:
        Hi, Wi, Ho, Wo = Hs, Ws, Hs, Ws
    elif mode == 1:
        Hi, Wi, Ho, Wo = 2 * Hs + 1, 2 * Ws + 1, Hs, Ws
    else:
        Hi, Wi, Ho, Wo = Hs, Ws, 2 * Hs + 1, 2 * Ws + 1
    x = round_tf32(torch.randn(B, Hi, Wi, Ci, device=cuda, generator=g))
    gy = round_tf32(torch.randn(B, Ho, Wo, Co, device=cuda, generator=g))
    res = []
    for impl in (2, 1):
        old = (ops.CONV_IMPL, ops.WGRAD_IMPL)
        ops.CONV_IMPL, ops.WGRAD_IMPL = (0, 2) if impl == 2 else (1, 1)
        try:
            res.append(ops._wgrad_raw(x, gy, k, mode, flip, transposed))
        finally:
            ops.CONV_IMPL, ops.WGRAD_IMPL = old
    torch.cuda.synchronize()
    assert res[0].shape == res[1].shape
    e = gu.rel_err(res[0].cpu().numpy(), res[1].cpu().numpy())
    assert e < 5e-5, e


# ------------------------------------------------------------------------------------------------ bf16x3 (compensated)
# The error-compensated mode (gifb200_conv2d / _wgrad impl 3): UNROUNDED fp32 operands, split into two bf16 terms by
# gifb200_split_bf16, hi*hi + hi*lo + lo*hi on bf16, fp32 accumulate.  Expected error ~2^-17 per operand (the dropped
# lo*lo term and the rounding of lo): the bar is 5e-5 against the exact-fp32 SIMT kernel on the same raw inputs -- 20x
# inside BASELINE.json's 1e-3 and 6x inside what tf32 can do (3e-4).
def test_split_bf16_planes(cuda):
    from gif_b200 import ops
    x = torch.randn(3, 5, 7, 32, device=cuda) * 3.0
    pl = ops._planes(x)
    assert pl.dtype == torch.bfloat16 and tuple(pl.shape) == (2, 3, 5, 7, 32)
    hi = x.to(torch.bfloat16)
    assert torch.equal(pl[0], hi)                                                   # round-to-nearest-even, like torch
    assert torch.equal(pl[1], (x - hi.float()).to(torch.bfloat16))
    rec = pl[0].float() + pl[1].float()
    assert float(((rec - x).abs() / x.abs().clamp_min(1e-30)).max()) < 2.0 ** -16
    assert ops._planes(x) is pl                                                     # cached under the version counter
    x.add_(1.0)
    assert ops._planes(x) is not pl


@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", CASES)
@pytest.mark.parametrize("flip,transposed", [(False, False), (True, True), (False, True)])
def test_bf16x3_conv_matches_exact_fp32(cuda, B, Hs, Ws, Ci, Co, k, mode, flip, transposed):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Hs + Ci + mode + 5)
    Hi, Wi = (Hs, Ws) if mode != 1 else (2 * Hs + 1, 2 * Ws + 1)
    x = torch.randn(B, Hi, Wi, Ci, device=cuda, generator=g)
    wshape = (k * k, Ci, Co) if transposed else (k * k, Co, Ci)
    w = torch.randn(*wshape, device=cuda, generator=g) / math.sqrt(Ci * k * k)
    y_x3 = run(x, w, k, mode, flip, transposed, 3)
    y_ref = run(x, w, k, mode, flip, transposed, 1)
    torch.cuda.synchronize()
    e = gu.rel_err(y_x3.cpu().numpy(), y_ref.cpu().numpy())
    assert 1e-8 < e < 5e-5, e        # > 1e-8: not the SIMT kernel again


@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", WG_CASES)
@pytest.mark.parametrize("flip,transposed", [(False, False), (True, True), (False, True)])
def test_bf16x3_wgrad_matches_exact_fp32(cuda, B, Hs, Ws, Ci, Co, k, mode, flip, transposed):
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 77 + Hs + Ci + mode + 5)
    if mode == 0:
        Hi, Wi, Ho, Wo = Hs, Ws, Hs, Ws
    elif mode == 1:
        Hi, Wi, Ho, Wo = 2 * Hs + 1, 2 * Ws + 1, Hs, Ws
    else:
        Hi, Wi, Ho, Wo = Hs, Ws, 2 * Hs + 1, 2 * Ws + 1
    x = torch.randn(B, Hi, Wi, Ci, device=cuda, generator=g)
    gy = torch.randn(B, Ho, Wo, Co, device=cuda, generator=g)
    res = []
    for impl in (3, 1):
        old = ops.CONV_IMPL
        ops.CONV_IMPL = impl
        try:
            assert lib_path(ops, B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl) == impl
            res.append(ops._wgrad_raw(x, gy, k, mode, flip, transposed))
        finally:
            ops.CONV_IMPL = old
    torch.cuda.synchronize()
    e = gu.rel_err(res[0].cpu().numpy(), res[1].cpu().numpy())
    assert 1e-8 < e < 5e-5, e


def lib_path(ops, B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl):
    from gif_b200._lib import lib
    return lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl)


def test_bf16x3_northstar_shape_sampled(cuda):
    """The north-star layer's contraction (128 -> 128, 3x3, 256^2; B = 4 here): bf16x3 and tf32 against exact fp32."""
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(99)
    x = torch.randn(4, 256, 256, 128, device=cuda, generator=g)
    w = torch.randn(9, 128, 128, device=cuda, generator=g) / math.sqrt(1152)
    y32 = run(x, w, 3, 0, False, False, 1)
    e3 = gu.rel_err(run(x, w, 3, 0, False, False, 3).cpu().numpy(), y32.cpu().numpy())
    et = gu.rel_err(run(round_tf32(x), w, 3, 0, False, False, 2).cpu().numpy(), y32.cpu().numpy())
    print(f"north-star contraction vs exact fp32: bf16x3 {e3:.2e}, tf32 {et:.2e}")
    assert e3 < 5e-5 and et < 1e-3
