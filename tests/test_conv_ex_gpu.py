"""GPU: gifb200_conv2d_ex (general-geometry convolution), gifb200_pool2d and gifb200_resize_bilinear against torch in float64.

Convolutions: every one of the 43 distinct FID Inception geometries at batch 2 and 33 (M = B*Ho*Wo not a multiple of the
128-row tile), plus odd non-square maps, batch 1, 1x1 maps, stride 2 on even and odd sizes and outputs written into a slice
of a wider tensor (guard values must survive outside [c0, c0+Co)).  impl 1 (exact fp32) against float64 F.conv2d at 2e-5,
impl 3 (bf16x3) against impl 1 at 5e-5, impl 2 (tf32, tf32-rounded inputs) against impl 1 at 2e-5 (the bar of
test_conv_tc_gpu.py), and repeated runs bitwise equal."""
import math

import pytest
import torch
import torch.nn.functional as F

from gif_b200 import ops
from gif_b200._lib import check, lib, ptr, stream
from gif_b200.inception import BLOCKS

pytestmark = pytest.mark.gpu

GUARD = -12345.0


def _map_size(name):
    """Input map size of a layer in the network at a 299^2 input."""
    sizes = {"Conv2d_1a": 299, "Conv2d_2a": 149, "Conv2d_2b": 147, "Conv2d_3b": 73, "Conv2d_4a": 73, "Mixed_5": 35,
             "Mixed_6a": 35, "Mixed_6": 17, "Mixed_7a": 17, "Mixed_7": 8}
    return next(v for k, v in sizes.items() if name.startswith(k))


def _geometries():
    """The distinct (Ci, Co, kh, kw, stride, pad_h, pad_w) of the network, each with the map size it first runs at."""
    seen = {}
    for mods in BLOCKS:
        for _, convs in mods:
            for name, *geo in convs:
                seen.setdefault(tuple(geo), _map_size(name))
    return [g + (h,) for g, h in seen.items()]


def run(x, w, kh, kw, stride, pad, impl, bias=None, out=None, c0=0, Cy=None):
    B, Hi, Wi, Ci = x.shape
    Co = w.shape[1]
    Ho, Wo = (Hi + 2 * pad[0] - kh) // stride + 1, (Wi + 2 * pad[1] - kw) // stride + 1
    if out is None:
        out = torch.full((B, Ho, Wo, Cy or Co), GUARD, device=x.device)
    xin = ops._planes(x) if impl == 3 else x
    nws = lib.gifb200_conv2d_ex_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad[0], pad[1], impl)
    ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=x.device)
    check(lib.gifb200_conv2d_ex(ptr(xin), ptr(w), ptr(out), B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad[0], pad[1],
                                out.shape[3], c0, impl, int(bias is not None), ptr(bias), 0, ptr(ws), nws, stream()),
          "gifb200_conv2d_ex")
    return out


def ref64(x, w, kh, kw, stride, pad, bias=None):
    T, Co, Ci = w.shape
    wt = w.double().reshape(kh, kw, Co, Ci).permute(2, 3, 0, 1)
    y = F.conv2d(x.double().permute(0, 3, 1, 2), wt, None if bias is None else bias.double(), stride=stride, padding=pad)
    if bias is not None:
        y = F.relu(y)
    return y.permute(0, 2, 3, 1)


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def inputs(B, H, W, Ci, Co, kh, kw, seed, rt=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, Ci, device="cuda", generator=g)
    w = torch.randn(kh * kw, Co, Ci, device="cuda", generator=g) / math.sqrt(Ci * kh * kw)
    if rt:
        x, w = ops._round_tf32_raw(x), ops._round_tf32_raw(w)
    return x, w


def _pad(c):
    return (c + 31) // 32 * 32


@pytest.mark.parametrize("B", [2, 33])
@pytest.mark.parametrize("g", _geometries(), ids=lambda g: "ci{}_co{}_{}x{}_s{}_p{}{}_h{}".format(*g))
def test_inception_geometries(cuda, g, B):
    ci, co, kh, kw, s, ph, pw, H = g
    ci, co = _pad(ci), _pad(co)
    if B == 33 and H > 73:
        H = 37                              # the stem's big maps at batch 33 only add run time: same geometry, smaller map
    x, w = inputs(B, H, H, ci, co, kh, kw, seed=sum(g) * 7 + B)
    bias = torch.randn(co, device=cuda) * 0.1
    want = ref64(x, w, kh, kw, s, (ph, pw), bias)
    y1 = run(x, w, kh, kw, s, (ph, pw), 1, bias)
    assert rel(y1, want) < 2e-5
    y2 = run(x, w, kh, kw, s, (ph, pw), 2, bias)
    assert rel(y2, y1) < 2e-5
    y3 = run(x, w, kh, kw, s, (ph, pw), 3, bias)
    assert rel(y3, y1) < 5e-5
    assert torch.equal(run(x, w, kh, kw, s, (ph, pw), 3, bias), y3)
    assert torch.equal(run(x, w, kh, kw, s, (ph, pw), 2, bias), y2)


@pytest.mark.parametrize("case", [
    # B, Hi, Wi, Ci, Co, kh, kw, stride, ph, pw
    (1, 13, 9, 64, 32, 3, 3, 1, 1, 1),
    (3, 23, 11, 32, 96, 1, 7, 1, 0, 3),
    (2, 1, 1, 64, 64, 1, 1, 1, 0, 0),         # 1x1 map
    (2, 1, 1, 32, 64, 3, 3, 1, 1, 1),         # 1x1 map, every tap but the centre in the padding
    (2, 16, 16, 32, 32, 3, 3, 2, 0, 0),       # stride 2, even size
    (2, 17, 15, 32, 64, 3, 3, 2, 0, 0),       # stride 2, odd sizes
    (2, 18, 18, 32, 32, 5, 5, 2, 2, 2),       # stride 2 with padding
    (5, 7, 29, 96, 128, 7, 1, 1, 3, 0),
    (2, 8, 8, 448, 384, 3, 3, 1, 1, 1),       # split-K
])
def test_odd_shapes(cuda, case):
    B, Hi, Wi, Ci, Co, kh, kw, s, ph, pw = case
    x, w = inputs(B, Hi, Wi, Ci, Co, kh, kw, seed=sum(case))
    want = ref64(x, w, kh, kw, s, (ph, pw))
    y1 = run(x, w, kh, kw, s, (ph, pw), 1)
    assert rel(y1, want) < 2e-5
    assert rel(run(x, w, kh, kw, s, (ph, pw), 2), y1) < 2e-5
    assert rel(run(x, w, kh, kw, s, (ph, pw), 3), y1) < 5e-5


@pytest.mark.parametrize("impl", [1, 2, 3])
def test_output_slice_and_guards(cuda, impl):
    B, H, Ci, Co, Cy, c0 = 3, 17, 64, 96, 256, 64
    x, w = inputs(B, H, H, Ci, Co, 3, 1, seed=7)
    bias = torch.randn(Co, device=cuda) * 0.1
    y = run(x, w, 3, 1, 1, (1, 0), impl, bias, Cy=Cy, c0=c0)
    want = ref64(x, w, 3, 1, 1, (1, 0), bias)
    assert rel(y[..., c0:c0 + Co], want) < (5e-5 if impl == 3 else 2e-5)
    assert bool((y[..., :c0] == GUARD).all()) and bool((y[..., c0 + Co:] == GUARD).all())


def test_padded_channels_are_exact_zeros(cuda):
    """Zero weights and zero bias in the padded output channels give exactly 0 after the ReLU (the next layer's padding)."""
    x, w = inputs(2, 35, 35, 64, 64, 1, 1, seed=9)
    w[:, 48:] = 0
    bias = torch.randn(64, device=cuda)
    bias[48:] = 0
    for impl in (1, 2, 3):
        y = run(x, w, 1, 1, 1, (0, 0), impl, bias)
        assert bool((y[..., 48:] == 0).all())


@pytest.mark.parametrize("op,stride,pad", [("max", 2, 0), ("max", 1, 1), ("avg", 1, 1)])
@pytest.mark.parametrize("hw", [(147, 147), (35, 35), (17, 17), (8, 8), (14, 9)])
def test_pool2d(cuda, op, stride, pad, hw):
    g = torch.Generator(device="cuda").manual_seed(hw[0] * 3 + stride)
    x = torch.randn(3, hw[0], hw[1], 64, device=cuda, generator=g)
    xd = x.double().permute(0, 3, 1, 2)
    if op == "max":
        want = F.max_pool2d(xd, 3, stride, pad)
    else:
        want = F.avg_pool2d(xd, 3, stride, pad, count_include_pad=False)
    want = want.permute(0, 2, 3, 1)
    out = torch.full(want.shape[:3] + (192,), GUARD, device=cuda)
    y = ops.pool2d(x, op, stride, pad, out=out, c0=96)
    got = y[..., 96:160]
    if op == "max":
        assert torch.equal(got.double(), want)
    else:
        assert rel(got, want) < 1e-6
    assert bool((y[..., :96] == GUARD).all()) and bool((y[..., 160:] == GUARD).all())


@pytest.mark.parametrize("size", [256, 512, 1024, 299, 73])
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
def test_resize_bilinear(cuda, size, layout):
    g = torch.Generator(device="cuda").manual_seed(size)
    x = torch.rand(2, 3, size, size, device=cuda, generator=g)
    if layout == "channels_last":
        x = x.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)          # NCHW view of channels-last storage
    want = 2 * F.interpolate(x.double(), size=(299, 299), mode="bilinear", align_corners=False) - 1
    y = ops.resize_bilinear(x, (299, 299), 32, 2.0, -1.0)
    assert y.shape == (2, 299, 299, 32)
    assert rel(y[..., :3].permute(0, 3, 1, 2), want) < 1e-6
    assert bool((y[..., 3:] == 0).all())


def test_forward_only(cuda):
    x = torch.zeros(1, 4, 4, 32, device=cuda, requires_grad=True)
    w = torch.zeros(1, 32, 32, device=cuda)
    with pytest.raises(RuntimeError, match="forward-only"):
        ops.conv2d_ex(x, w, 1, 1)
    with pytest.raises(RuntimeError, match="forward-only"):
        ops.pool2d(x, "max", 2, 0)
