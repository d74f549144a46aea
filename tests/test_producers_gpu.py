"""GPU: the fused operand producers on the paths the model takes.

* bf16x3 planes: ``gifb200_tail_bwd_planes`` (C % 32 == 0, P >= 256), ``gifb200_tail_bwd2``'s ``ggy_planes`` and
  ``gifb200_split_bf16`` with a modulation vector, called with every NULL combination ``ops`` passes.  The planes must be
  bitwise the round-to-nearest-even split of the fp32 value (hi = bf16(v), lo = bf16(v - hi)) and every fp32 output
  within 2e-5 of float64 torch.
* tf32 rounding: for every producer with a ``round_tf32`` flag, the rt=1 output is bitwise the round-to-nearest-away
  tf32 rounding of the rt=0 output, ``(bits + 0x1000) & ~0x1FFF`` on the magnitude -- on exact ties, values near the
  float32 maximum, the vectorised widths and the scalar tails."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 2e-5


def _ops():
    from gif_b200 import ops
    return ops


def _p(t):
    return None if t is None else t.data_ptr()


def _rand(shape, seed, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=g) * (hi - lo) + lo).cuda()


def _rne_split(v):
    hi = v.bfloat16()
    return hi, (v - hi.float()).bfloat16()


def _assert_planes(pl, v, what):
    hi, lo = _rne_split(v)
    assert pl.dtype == torch.bfloat16
    assert torch.equal(pl[0].view(torch.int16), hi.view(torch.int16)), f"{what}: hi plane"
    assert torch.equal(pl[1].view(torch.int16), lo.view(torch.int16)), f"{what}: lo plane"


def _close(got, want, what):
    want = want.double()
    err = float((got.double() - want).abs().max()) / max(float(want.abs().max()), 1e-30)
    assert err < TOL, f"{what}: rel err {err:.2e} vs float64"


def _planes_like(t):
    return torch.empty((2,) + tuple(t.shape), dtype=torch.bfloat16, device=t.device)


SHAPES = [(2, 256, 32), (2, 300, 64), (1, 289, 512), (2, 256, 512)]     # P >= 256, ragged P included


# --------------------------------------------------------------------------------------------- tail_bwd_planes
@pytest.mark.parametrize("B,P,C", SHAPES)
@pytest.mark.parametrize("want_b", [False, True])
def test_tail_bwd_planes_conv_bias_act(cuda, B, P, C, want_b):
    """The first-order backward of _Conv's fused epilogue: only the planes of gt (no fp32 gt), acc = y, no d, optional
    bias gradient."""
    ops = _ops()
    rows, slope, gain = B * P, 0.2, 2 ** 0.5
    gy, y = _rand((rows, C), 1), _rand((rows, C), 2)
    gb = torch.full((C,), float("nan"), device=cuda) if want_b else None
    pl = _planes_like(gy)
    ops.check(ops.lib.gifb200_tail_bwd_planes(_p(gy), _p(y), _p(y), None, None, None, _p(gb), None, 1, rows, C, slope,
                                              gain, _p(pl), None, ops.stream()), "tail_bwd_planes")
    m = torch.where(y > 0, 1.0, slope)
    _assert_planes(pl, gy * gain * m, "gt")                          # fp32 gt: (gy*gain)*m, the kernel's order
    if want_b:
        _close(gb, (gy.double() * gain * m.double()).sum(0), "gb")


_BIAS_ACT_CASES = [(rs, add, b, d) for rs in (False, True) for add in (False, True) for b in (False, True)
                   for d in ((False, True) if rs else (False,))]


@pytest.mark.parametrize("B,P,C", SHAPES)
@pytest.mark.parametrize("rowscale,has_add,want_b,want_d", _BIAS_ACT_CASES)
def test_tail_bwd_planes_bias_act(cuda, B, P, C, rowscale, has_add, want_b, want_d):
    """_BiasAct's first-order backward in bf16x3: fp32 gt (and gacc with a rowscale) plus their planes in the same pass."""
    ops = _ops()
    slope, gain = 0.2, 2 ** 0.5
    gy, y, x = _rand((B, P, C), 3), _rand((B, P, C), 4), _rand((B, P, C), 5)
    d = _rand((B, C), 6, 0.5, 1.5) if rowscale else None
    gt = torch.empty_like(gy)
    gacc = torch.empty_like(gy) if rowscale else None
    gb = torch.empty(C, device=cuda) if want_b else None
    gd = torch.empty((B, C), device=cuda) if want_d else None
    pt = _planes_like(gy) if has_add else None
    pa = _planes_like(gy) if rowscale else None
    ops.check(ops.lib.gifb200_tail_bwd_planes(_p(gy), _p(y), _p(x), _p(d), _p(gt), _p(gacc), _p(gb), _p(gd), B, P, C,
                                              slope, gain, _p(pt), _p(pa), ops.stream()), "tail_bwd_planes")
    m64 = torch.where(y > 0, 1.0, slope).double() * gain
    gt64 = gy.double() * m64
    _close(gt, gt64, "gt")
    if pt is not None:
        _assert_planes(pt, gt, "gt planes")
    if rowscale:
        _close(gacc, gt64 * d.double()[:, None, :], "gacc")
        _assert_planes(pa, gacc, "gacc planes")
    if want_b:
        _close(gb, gt64.sum((0, 1)), "gb")
    if want_d:
        _close(gd, (gt64 * x.double()).sum(1), "gd")


@pytest.mark.parametrize("B,P,C", SHAPES)
def test_tail_bwd_planes_second_order_node(cuda, B, P, C):
    """_TailBwdCG.forward (path-length pass): gacc with its planes and gd; no gt, no bias gradient."""
    ops = _ops()
    slope, gain = 0.2, 2 ** 0.5
    gy, y, acc = _rand((B, P, C), 7), _rand((B, P, C), 8), _rand((B, P, C), 9)
    d = _rand((B, C), 10, 0.5, 1.5)
    gacc, gd, pa = torch.empty_like(gy), torch.empty((B, C), device=cuda), _planes_like(gy)
    ops.check(ops.lib.gifb200_tail_bwd_planes(_p(gy), _p(y), _p(acc), _p(d), None, _p(gacc), None, _p(gd), B, P, C,
                                              slope, gain, None, _p(pa), ops.stream()), "tail_bwd_planes")
    gt64 = gy.double() * torch.where(y > 0, 1.0, slope).double() * gain
    _close(gacc, gt64 * d.double()[:, None, :], "gacc")
    _assert_planes(pa, gacc, "gacc planes")
    _close(gd, (gt64 * acc.double()).sum(1), "gd")


# --------------------------------------------------------------------------------------------- tail_bwd2 ggy planes
_BWD2_CASES = [(gg, ggd, gx2, gdd) for gg in (False, True) for ggd in (False, True) if gg or ggd
               for gx2 in ((False, True) if ggd else (False,)) for gdd in ((False, True) if gg else (False,))]


@pytest.mark.parametrize("B,P,C", SHAPES)
@pytest.mark.parametrize("has_gg,has_ggd,want_gx2,want_gdd", _BWD2_CASES)
def test_tail_bwd2_ggy_planes(cuda, B, P, C, has_gg, has_ggd, want_gx2, want_gdd):
    """_TailBwdCG.backward of the modulation node (y NULL: m = 1) in bf16x3: ggy and its planes in one pass."""
    ops = _ops()
    gy, acc = _rand((B, P, C), 11), _rand((B, P, C), 12)
    d = _rand((B, C), 13, 0.5, 1.5)
    gg = _rand((B, P, C), 14) if has_gg else None
    ggd = _rand((B, C), 15) if has_ggd else None
    ggy, pp = torch.empty_like(gy), _planes_like(gy)
    gx2 = torch.empty_like(gy) if want_gx2 else None
    gdd = torch.full((B, C), float("nan"), device=cuda) if want_gdd else None
    ops.check(ops.lib.gifb200_tail_bwd2(_p(gg), _p(ggd), _p(gy), None, _p(acc), _p(d), _p(ggy), _p(gx2), _p(gdd), B, P, C,
                                        0.2, 2 ** 0.5, _p(pp), ops.stream()), "tail_bwd2")
    want = torch.zeros_like(gy, dtype=torch.float64)
    if has_gg:
        want += gg.double() * d.double()[:, None, :]
    if has_ggd:
        want += ggd.double()[:, None, :] * acc.double()
    _close(ggy, want, "ggy")
    _assert_planes(pp, ggy, "ggy planes")
    if want_gx2:
        _close(gx2, gy.double() * ggd.double()[:, None, :], "gx2")
    if want_gdd:
        _close(gdd, (gg.double() * gy.double()).sum(1), "gdd")


# --------------------------------------------------------------------------------------------- split_bf16
@pytest.mark.parametrize("B,P,C", SHAPES + [(2, 81, 20), (3, 7, 4)])
@pytest.mark.parametrize("with_s", [False, True])
def test_split_bf16(cuda, B, P, C, with_s):
    """The operand split, plain (``ops._planes``) and fused with the modulation (``_ModConvX3``): the split of x*s in fp32."""
    ops = _ops()
    x = _rand((B, P, C), 16, -3.0, 3.0)
    s = _rand((B, C), 17, 0.1, 2.0) if with_s else None
    pl = _planes_like(x)
    ops.check(ops.lib.gifb200_split_bf16(_p(x), _p(s), _p(pl), B, P, C, ops.stream()), "split_bf16")
    _assert_planes(pl, x * s[:, None, :] if with_s else x, "planes")


# --------------------------------------------------------------------------------------------- tf32 rounding
def _rna_tf32(a):
    """Round-to-nearest-away to tf32 (10 explicit mantissa bits), on the magnitude bits."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    mag = ((u & np.uint32(0x7FFFFFFF)) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    return ((u & np.uint32(0x80000000)) | mag).view(np.float32)


def _edge_values(shape, seed):
    """Random values with a third replaced by exact ties (low 13 bits 0x1000) and some by values within a tf32 step of
    the float32 maximum (which round up to infinity or down to the largest tf32)."""
    rng = np.random.default_rng(seed)
    v = rng.uniform(-4, 4, size=shape).astype(np.float32)
    u = v.view(np.uint32)
    ties = rng.random(shape) < 0.35
    u[ties] = (u[ties] & np.uint32(0xFFFFE000)) | np.uint32(0x1000)
    big = rng.random(shape) < 0.05
    top = np.array([0x7F7FFFFF, 0x7F7FF000, 0x7F7FEFFF, 0x7F7FE000, 0x7F7FD000, 0x7F000000], np.uint32)
    u[big] = top[rng.integers(0, len(top), int(big.sum()))] | (rng.integers(0, 2, int(big.sum())).astype(np.uint32) << 31)
    return torch.from_numpy(u.view(np.float32).copy()).cuda()


def _assert_rna(y1, y0, what):
    a0, a1 = y0.cpu().numpy().ravel(), y1.cpu().numpy().ravel()
    assert np.isfinite(a0).all()
    want = _rna_tf32(a0)
    bad = np.flatnonzero(want.view(np.uint32) != a1.view(np.uint32))
    assert bad.size == 0, (f"{what}: {bad.size} of {a0.size} values not rounded to nearest-away tf32, e.g. "
                           f"{a0[bad[0]]!r} -> {a1[bad[0]]!r} (want {want[bad[0]]!r})")


def _both(fn):
    return fn(False), fn(True)


ELEM_SHAPES = [(2, 81, 32), (2, 81, 20), (2, 9, 5)]               # float4 path, scalar tails


@pytest.mark.parametrize("B,P,C", ELEM_SHAPES)
@pytest.mark.parametrize("edge", [True, False])
def test_round_tf32_elementwise_producers(cuda, B, P, C, edge):
    ops = _ops()
    x = _edge_values((B, P, C), 20) if edge else _rand((B, P, C), 20, -3, 3)
    y = _rand((B, P, C), 21)
    s = torch.ones((B, C), device=cuda) if edge else _rand((B, C), 22, 0.5, 1.5)
    bias = None if edge else _rand((C,), 23)
    slope, gain = (1.0, 1.0) if edge else (0.2, 2 ** 0.5)
    y_pos = y.abs() + 0.5 if edge else y                               # edge: m = 1, the outputs are the inputs
    n = x.numel()

    def bias_act(rt):
        out = torch.empty_like(x)
        ops.check(ops.lib.gifb200_bias_act(_p(x), None if edge else _p(s), None, _p(bias), _p(out), B, P, C, slope, gain,
                                           int(rt), ops.stream()), "bias_act")
        return out

    def act_bwd(rt):
        out = torch.empty_like(x)
        ops.check(ops.lib.gifb200_act_bwd(_p(x), _p(y_pos), _p(out), n, slope, gain, int(rt), ops.stream()), "act_bwd")
        return out

    def chan_scale(rt):
        out = torch.empty_like(x)
        ops.check(ops.lib.gifb200_chan_scale(_p(x), _p(s), _p(out), B, P, C, int(rt), ops.stream()), "chan_scale")
        return out

    def axpby(rt):
        out = torch.empty_like(x)
        b, beta = (None, 0.0) if edge else (y, 0.7)
        ops.check(ops.lib.gifb200_axpby(_p(x), _p(b), _p(out), n, 1.0 if edge else 0.7, beta, int(rt), ops.stream()),
                  "axpby")
        return out

    def tail_bwd(rt):
        gt, gacc = torch.empty_like(x), torch.empty_like(x)
        d = s
        ops.check(ops.lib.gifb200_tail_bwd(_p(x), _p(y_pos), _p(y), _p(d), _p(gt), _p(gacc), None, None, B, P, C, slope,
                                           gain, int(rt), ops.stream()), "tail_bwd")
        return torch.stack([gt, gacc])

    for name, fn in [("bias_act", bias_act), ("act_bwd", act_bwd), ("chan_scale", chan_scale), ("axpby", axpby),
                     ("tail_bwd", tail_bwd)]:
        y0, y1 = _both(fn)
        _assert_rna(y1, y0, name)


@pytest.mark.parametrize("C", [32, 20, 5])
@pytest.mark.parametrize("up,down,kw", [(1, 1, 1), (1, 1, 4), (2, 1, 4), (1, 2, 4)])
def test_round_tf32_upfirdn2d(cuda, C, up, down, kw):
    ops = _ops()
    B, H = 2, 11
    x = _edge_values((B, H, H, C), 30) if kw == 1 else _rand((B, H, H, C), 30)
    k = torch.ones((1, 1), device=cuda) if kw == 1 else torch.outer(*(2 * [torch.tensor([1.0, 3.0, 3.0, 1.0])])).cuda() / 16
    pad = (0, 0) if kw == 1 else (2, 1)
    y0, y1 = (ops.upfirdn2d(x, k, up, down, pad, rt=rt) for rt in (False, True))
    _assert_rna(y1, y0, "upfirdn2d")


@pytest.mark.parametrize("mode", ["tf32", "bf16x3", "fp32"])
@pytest.mark.parametrize("B,H,Ci,Co", [(2, 4, 512, 512), (2, 32, 64, 128), (2, 7, 20, 5)])
def test_round_tf32_conv_epilogue(cuda, mode, B, H, Ci, Co):
    """The fused conv epilogue's rounding: direct (non-split tiles, SIMT) and through the split-K reduction (4x4 at 512
    channels: the tiles cannot fill the machine)."""
    ops = _ops()
    old = ops.get_precision()
    ops.set_precision(mode)
    try:
        x = _rand((B, H, H, Ci), 40)
        w = _rand((9, Co, Ci), 41, -0.05, 0.05)
        bias = _rand((Co,), 42)
        nws = ops.lib.gifb200_conv2d_workspace_bytes(B, H, H, Ci, H, H, Co, 3, ops.S1, 0, ops.CONV_IMPL)
        if mode != "fp32" and Ci >= 32:
            assert nws > 0                                        # the tensor-core path is the one under test
        y0, y1 = (ops._conv_raw(x, w, 3, ops.S1, False, False, (H, H), (bias, 0.2, 2 ** 0.5, rt))[0] for rt in (0, 1))
    finally:
        ops.set_precision(old)
    _assert_rna(y1, y0, f"conv epilogue [{mode}]")


@pytest.mark.parametrize("C", [32, 20, 5])
@pytest.mark.parametrize("op,stride,pad", [("max", 1, 1), ("max", 2, 0), ("avg", 1, 1), ("avg", 2, 1)])
def test_round_tf32_pool2d(cuda, C, op, stride, pad):
    ops = _ops()
    x = _edge_values((2, 9, 9, C), 50) if op == "max" else _rand((2, 9, 9, C), 50)
    y0, y1 = (ops.pool2d(x, op, stride, pad, round_tf32=rt) for rt in (False, True))
    _assert_rna(y1, y0, f"pool2d {op}")


@pytest.mark.parametrize("size,channels", [((13, 17), 32), ((8, 8), 5), ((40, 24), 20)])
def test_round_tf32_resize_bilinear(cuda, size, channels):
    ops = _ops()
    x = _rand((2, 3, 19, 23), 60)
    y0, y1 = (ops.resize_bilinear(x, size, channels, 2.0, -1.0, round_tf32=rt) for rt in (False, True))
    _assert_rna(y1, y0, "resize_bilinear")
    ref = F.interpolate(x.double(), size, mode="bilinear", align_corners=False) * 2.0 - 1.0
    _close(y0[..., :3], ref.permute(0, 2, 3, 1), "resize_bilinear vs torch")


@pytest.mark.parametrize("mode", ["tf32", "bf16x3", "fp32"])
@pytest.mark.parametrize("B,H,Ci,Co,kh,kw,stride,pad", [(2, 17, 64, 64, 3, 3, 1, (1, 1)), (2, 8, 64, 32, 1, 7, 1, (0, 3)),
                                                        (2, 9, 5, 20, 3, 3, 2, (0, 0))])
def test_round_tf32_conv2d_ex(cuda, mode, B, H, Ci, Co, kh, kw, stride, pad):
    ops = _ops()
    old = ops.get_precision()
    ops.set_precision(mode)
    try:
        x = _rand((B, H, H, Ci), 70)
        w = _rand((kh * kw, Co, Ci), 71, -0.1, 0.1)
        bias = _rand((Co,), 72)
        with torch.no_grad():
            y0, y1 = (ops.conv2d_ex(x, w, kh, kw, stride, pad, bias, relu=True, round_tf32=rt) for rt in (False, True))
    finally:
        ops.set_precision(old)
    _assert_rna(y1, y0, f"conv2d_ex [{mode}]")
