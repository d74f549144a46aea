"""GPU: the narrow (M = 64) variant of the tensor-core weight gradient -- small side of 64 channels (S1 / S2 / T2, 3x3; S1
1x1) or 32 channels (S1 1x1, up to 64 big channels), the shapes of the 512^2 / 1024^2 layers.  tf32 against the exact-fp32 SIMT kernel on
tf32-rounded inputs, bf16x3 against exact fp32 on raw inputs (the bars of test_conv_tc_gpu.py), bitwise repeatable."""
import pytest
import torch

import golden_util as gu

pytestmark = pytest.mark.gpu

CASES = [
    # (B, Hs, Ws, Ci, Co, k, mode)   Hs/Ws = SITE grid (output for S1/S2, input for T2)
    # the layers themselves (batch 1)
    (1, 512, 512, 64, 64, 3, 0),     # G progression.7.st_cv2; D ResBlock(64->128).conv1 @512
    (1, 512, 512, 32, 64, 3, 0),     # G noise conv 24->64 (input padded to 32)
    (1, 512, 512, 64, 32, 3, 2),     # G progression.8.st_cv1 (T2 to 1025^2)
    (1, 512, 512, 32, 64, 1, 0),     # D 512 stem (padded to 32); D 1024 ResBlock(32->64).skip
    (1, 1024, 1024, 32, 32, 1, 0),   # D 1024 stem
    (1, 512, 512, 32, 64, 3, 1),     # D 1024 ResBlock(32->64).conv2 (S2 from 1025^2)
    # small variants: odd batch, narrow images (multi-row boxes), Cb of 32 / 64 / 128
    (3, 8, 8, 64, 64, 3, 0), (6, 4, 4, 128, 64, 3, 0), (1, 32, 64, 32, 64, 3, 0), (3, 16, 16, 32, 64, 1, 0),
    (2, 8, 8, 32, 32, 1, 0), (3, 4, 8, 64, 32, 1, 0), (3, 16, 16, 64, 64, 1, 0),
    (3, 8, 8, 64, 64, 3, 1), (2, 16, 32, 128, 64, 3, 1), (1, 64, 64, 32, 64, 3, 1),
    (3, 8, 8, 64, 64, 3, 2), (2, 16, 16, 64, 128, 3, 2), (1, 64, 64, 64, 32, 3, 2),
]


def grids(Hs, Ws, mode):
    if mode == 0:
        return Hs, Ws, Hs, Ws
    if mode == 1:
        return 2 * Hs + 1, 2 * Ws + 1, Hs, Ws
    return Hs, Ws, 2 * Hs + 1, 2 * Ws + 1


def wgrad(x, gy, k, mode, flip, transposed, impl):
    from gif_b200 import ops
    old = (ops.CONV_IMPL, ops.WGRAD_IMPL)
    ops.CONV_IMPL, ops.WGRAD_IMPL = {1: (1, 1), 2: (0, 2), 3: (3, 3)}[impl]
    try:
        return ops._wgrad_raw(x, gy, k, mode, flip, transposed)
    finally:
        ops.CONV_IMPL, ops.WGRAD_IMPL = old


@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", CASES)
@pytest.mark.parametrize("flip,transposed", [(False, False), (True, True), (False, True)])
@pytest.mark.parametrize("impl", [2, 3])
def test_narrow_wgrad(cuda, B, Hs, Ws, Ci, Co, k, mode, flip, transposed, impl):
    from gif_b200 import ops
    from gif_b200._lib import lib
    Hi, Wi, Ho, Wo = grids(Hs, Ws, mode)
    assert lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl) == impl
    g = torch.Generator(device="cuda").manual_seed(B * 77 + Hs + Ci + Co + mode + k + impl)
    x = torch.randn(B, Hi, Wi, Ci, device=cuda, generator=g)
    gy = torch.randn(B, Ho, Wo, Co, device=cuda, generator=g)
    if impl == 2:
        x, gy = ops._round_tf32_raw(x), ops._round_tf32_raw(gy)
    got = wgrad(x, gy, k, mode, flip, transposed, impl)
    ref = wgrad(x, gy, k, mode, flip, transposed, 1)
    again = wgrad(x, gy, k, mode, flip, transposed, impl)
    torch.cuda.synchronize()
    assert got.shape == ref.shape
    e = gu.rel_err(got.cpu().numpy(), ref.cpu().numpy())
    assert (e < 5e-5) and (impl == 2 or e > 1e-8), e          # bf16x3: > 1e-8, not the SIMT kernel again
    assert torch.equal(got, again)                              # fixed reduction order


def test_narrow_wgrad_runs_the_tensor_core_kernel(cuda):
    """The 512^2 64 -> 64 layer launches wgrad_tc_kernel and no SIMT weight-gradient kernel."""
    from test_layer_shapes_gpu import kernel_names
    x = torch.randn(1, 512, 512, 64, device=cuda)
    gy = torch.randn(1, 512, 512, 64, device=cuda)
    wgrad(x, gy, 3, 0, False, False, 3)
    torch.cuda.synchronize()
    # a profiling window with CUDA activity alone now and then holds no kernel records: profile again (see kernel_names)
    names = kernel_names(lambda: wgrad(x, gy, 3, 0, False, False, 3), lambda ns: any("wgrad_tc_kernel" in n for n in ns))
    assert any("wgrad_tc_kernel" in n for n in names), names
    assert not any("wgrad_simt_kernel" in n for n in names), names
