"""GPU parity tests of the individual operators: the CUDA path (through the C ABI, gif_b200.ops / gif_b200.model)
against (a) the golden vectors produced by the UNMODIFIED reference modules (tests/golden/*.npz, written by
oracle/make_golden.py) and (b) the oracle restatement evaluated live on the CPU on the same seeded inputs.

Tolerances (norm-wise relative error max|a-b|/max|b|, golden_util.rel_err):
  * fp32 mode (SIMT kernels):   2e-5  -- fp32 reassociation only
  * tf32 mode (wgmma kernels): 1e-3 -- the bar stated in BASELINE.json ("within 1e-3 relative fp32")
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu
from oracle import stylegan2_oracle as O

pytestmark = pytest.mark.gpu
TOL32 = 2e-5


def nhwc(t, dev):
    return t.permute(0, 2, 3, 1).contiguous().to(dev)


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous().cpu()


def close(a, b, tol, what=""):
    e = gu.rel_err(a.detach().cpu().double().numpy() if torch.is_tensor(a) else a,
                   b.detach().cpu().double().numpy() if torch.is_tensor(b) else b)
    assert e < tol, f"{what}: rel err {e:.3e} >= {tol}"
    return e


# ------------------------------------------------------------------------------------------------ upfirdn2d
UPFIRDN_CASES = [(1, 1, (1, 1), 4.0), (1, 1, (2, 2), 1.0), (1, 1, (1, 1), 1.0), (2, 1, (2, 1), 4.0),
                 (1, 2, (1, 1), 1.0), (1, 2, (0, 0), 1.0), (1, 1, (-1, 0), 1.0)]


def test_upfirdn2d_golden(cuda):
    from gif_b200.model import stylegan2_common_layers as cl
    g = gu.load_golden("ops.npz")
    for ci, (up, down, pad, gain) in enumerate(UPFIRDN_CASES):
        for si, (h, w) in enumerate([(9, 9), (8, 5), (17, 33)]):
            x = gu.randn((2, 3, h, w), 10 + ci * 7 + si)
            y = cl.upfirdn2d(x.to(cuda), gu.blur_kernel(gain).to(cuda), up=up, down=down, pad=pad)
            assert tuple(y.shape) == g[f"upfirdn_{ci}_{si}"].shape
            close(y, g[f"upfirdn_{ci}_{si}"], TOL32, f"upfirdn2d case {ci},{si}")
    ka = torch.from_numpy(g["upfirdn_asym_k"])
    y = cl.upfirdn2d(gu.randn((1, 2, 7, 6), 98).to(cuda), ka.to(cuda), up=2, down=1, pad=(2, 1))
    close(y, g["upfirdn_asym"], TOL32, "upfirdn2d asymmetric kernel (flip convention)")


@pytest.mark.parametrize("c", [4, 32, 5])
@pytest.mark.parametrize("up,down,pad", [(1, 1, (2, 2)), (2, 1, (2, 1)), (1, 2, (1, 1)), (1, 1, (1, 1))])
def test_upfirdn2d_backward_and_double_backward(cuda, fp32_mode, c, up, down, pad):
    """vectorised (C%4==0) and scalar paths; first and second derivative against the oracle's autograd."""
    from gif_b200 import ops
    k = gu.randn((4, 4), 5)      # asymmetric: the adjoint must flip
    x = gu.randn((2, c, 10, 7), 6)
    xg = nhwc(x, cuda).requires_grad_(True)
    y = ops.upfirdn2d(xg, k.to(cuda), up, down, pad)
    xo = x.clone().requires_grad_(True)
    yo = O.upfirdn2d(xo, k, up, down, pad)
    close(nchw(y), yo, TOL32, "fwd")
    gy = gu.randn(tuple(yo.shape), 7)
    (gx,) = torch.autograd.grad(y, xg, nhwc(gy, cuda), create_graph=True)
    (gxo,) = torch.autograd.grad(yo, xo, gy, create_graph=True)
    close(nchw(gx), gxo, TOL32, "bwd")
    v = gu.randn(tuple(x.shape), 8)
    # gx is linear in gy only; differentiate <gx, v> w.r.t. the upstream seed through a fresh graph
    gys = nhwc(gy, cuda).requires_grad_(True)
    (gx2,) = torch.autograd.grad(ops.upfirdn2d(xg, k.to(cuda), up, down, pad), xg, gys, create_graph=True)
    (gg,) = torch.autograd.grad((gx2 * nhwc(v, cuda)).sum(), gys)
    close(nchw(gg), O.upfirdn2d(v, k, up, down, pad), TOL32, "double bwd")


@pytest.mark.parametrize("c,h,w", [(32, 21, 19), (64, 16, 40), (32, 9, 8)])
@pytest.mark.parametrize("pad", [(1, 1), (0, 0), (2, 2), (2, 1)])
def test_upfirdn2d_down2_tiled_kernel(cuda, fp32_mode, c, h, w, pad):
    """the shared-memory tiled decimating FIR (C % 32 == 0, 4x4, down 2): ragged tile edges, every pad the model uses,
    asymmetric kernel; forward vs the oracle and, through the up=2 call whose adjoint it is, the flipped variant."""
    from gif_b200 import ops
    k = gu.randn((4, 4), 15)
    x = gu.randn((2, c, h, w), 16)
    y = ops.upfirdn2d(nhwc(x, cuda), k.to(cuda), 1, 2, pad)
    close(nchw(y), O.upfirdn2d(x, k, 1, 2, pad), TOL32, "down2 fwd")
    # adjoint of up=2 (runs the same kernel with flip=1 and pad' = k-1-pad)
    xs = gu.randn((2, c, h // 2 + 1, w // 2 + 1), 17)
    xg = nhwc(xs, cuda).requires_grad_(True)
    yu = ops.upfirdn2d(xg, k.to(cuda), 2, 1, pad)
    xo = xs.clone().requires_grad_(True)
    yo = O.upfirdn2d(xo, k, 2, 1, pad)
    close(nchw(yu), yo, TOL32, "up2 fwd")
    gy = gu.randn(tuple(yo.shape), 18)
    (gx,) = torch.autograd.grad(yu, xg, nhwc(gy, cuda))
    (gxo,) = torch.autograd.grad(yo, xo, gy)
    close(nchw(gx), gxo, TOL32, "up2 bwd (down2 kernel, flipped)")


@pytest.mark.parametrize("c,h,w", [(32, 21, 19), (64, 16, 40), (32, 5, 6)])
@pytest.mark.parametrize("pad", [(1, 1), (2, 2), (2, 1)])
@pytest.mark.parametrize("kind", ["blur", "random"])
def test_upfirdn2d_blur_tiled_kernel(cuda, fp32_mode, c, h, w, pad, kind):
    """the pipelined shared-memory 4x4 FIR (C % 32 == 0, up = down = 1): the rank-1 fast path taken for the model's
    blur kernel and the general path (random asymmetric kernel), ragged tiles, forward and adjoint (flip)."""
    from gif_b200 import ops
    k = gu.blur_kernel(4.0) if kind == "blur" else gu.randn((4, 4), 25)
    x = gu.randn((2, c, h, w), 26)
    xg = nhwc(x, cuda).requires_grad_(True)
    y = ops.upfirdn2d(xg, k.to(cuda), 1, 1, pad)
    xo = x.clone().requires_grad_(True)
    yo = O.upfirdn2d(xo, k, 1, 1, pad)
    close(nchw(y), yo, TOL32, "blur fwd")
    gy = gu.randn(tuple(yo.shape), 27)
    (gx,) = torch.autograd.grad(y, xg, nhwc(gy, cuda))
    (gxo,) = torch.autograd.grad(yo, xo, gy)
    close(nchw(gx), gxo, TOL32, "blur bwd")


# ------------------------------------------------------------------------------------------------ small ops
def test_small_ops_golden(cuda):
    from gif_b200.model import stylegan2_common_layers as cl
    g = gu.load_golden("ops.npz")
    m = cl.FusedLeakyReLU(5).to(cuda)
    m.bias.data = gu.randn((1, 5, 1, 1), 3).to(cuda)
    close(m(gu.randn((2, 5, 4, 4), 4).to(cuda)), g["lrelu"], 1e-6, "FusedLeakyReLU")
    for tag, kw in (("act", dict(lr_mul=0.01, activation="fused_lrelu")), ("plain", dict(bias_init=1))):
        m = cl.EqualLinear(24, 16, **kw).to(cuda)
        m.weight.data = (gu.randn((16, 24), 5) * (100.0 if tag == "act" else 1.0)).to(cuda)
        m.bias.data = gu.randn((16,), 6).to(cuda)
        close(m(gu.randn((3, 24), 7).to(cuda)), g[f"linear_{tag}"], TOL32, f"EqualLinear[{tag}]")


@pytest.mark.parametrize("tag,k,s,p,hw", [("k1", 1, 1, 0, 8), ("k3s1", 3, 1, 1, 8), ("k3s2", 3, 2, 0, 9), ("k1s2", 1, 2, 0, 7)])
def test_equal_conv2d_golden(cuda, fp32_mode, tag, k, s, p, hw):
    from gif_b200.model import stylegan2_common_layers as cl
    g = gu.load_golden("ops.npz")
    m = cl.EqualConv2d(6, 10, k, stride=s, padding=p, bias=False).to(cuda)
    m.weight.data = gu.randn((10, 6, k, k), 8).to(cuda)
    y = m(gu.randn((2, 6, hw, hw), 9).to(cuda))
    assert tuple(y.shape) == g[f"conv_{tag}"].shape
    close(y, g[f"conv_{tag}"], TOL32, f"EqualConv2d[{tag}]")


def test_unsupported_conv_raises(cuda):
    from gif_b200.model import stylegan2_common_layers as cl
    with pytest.raises(NotImplementedError):
        cl.EqualConv2d(4, 4, 3, stride=1, padding=0).to(cuda)(torch.zeros(1, 4, 8, 8, device=cuda))


def test_cpu_tensor_raises():
    """No CPU fallback: the product path must fail loudly."""
    from gif_b200 import ops
    from gif_b200._lib import GifB200Error
    with pytest.raises(GifB200Error):
        ops.bias_act(torch.zeros(1, 2, 2, 4), None)


# ------------------------------------------------------------------------------------------------ conv primitives
def _ref_conv(x, w_tap, k, mode):
    """torch CPU reference of the three modes from a tap-major (T,Co,Ci) weight."""
    T, co, ci = w_tap.shape
    w = w_tap.reshape(k, k, co, ci).permute(2, 3, 0, 1)
    if mode == 0:
        return F.conv2d(x, w, padding=k // 2)
    if mode == 1:
        return F.conv2d(x, w, stride=2)
    return F.conv_transpose2d(x, w.transpose(0, 1), stride=2)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("ci,co", [(6, 12), (32, 16), (9, 128), (70, 66)])
def test_conv_modes_simt(cuda, fp32_mode, mode, k, ci, co):
    """forward, input gradient (adjoint call on the same weight buffer), weight gradient, and both second
    derivatives of the bilinear map, for every mode; ragged channel counts exercise the tile edges."""
    from gif_b200 import ops
    hi = 9 if mode != 2 else 5
    x = gu.randn((2, ci, hi, hi + 2), 1)
    w = gu.randn((k * k, co, ci), 2) / math.sqrt(ci * k * k)
    xg = nhwc(x, cuda).requires_grad_(True)
    wg = w.to(cuda).requires_grad_(True)
    y = ops.conv2d(xg, wg, k, mode)
    xo, wo = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    yo = _ref_conv(xo, wo, k, mode)
    assert tuple(nchw(y).shape) == tuple(yo.shape)
    close(nchw(y), yo, TOL32, "fwd")
    gy = gu.randn(tuple(yo.shape), 3)
    gx, gw = torch.autograd.grad(y, [xg, wg], nhwc(gy, cuda), create_graph=True)
    gxo, gwo = torch.autograd.grad(yo, [xo, wo], gy, create_graph=True)
    close(nchw(gx), gxo, TOL32, "dgrad")
    close(gw, gwo, TOL32, "wgrad")
    vx, vw = gu.randn(tuple(x.shape), 4), gu.randn(tuple(w.shape), 5)
    ggx, ggw = torch.autograd.grad((gx * nhwc(vx, cuda)).sum() + (gw * vw.to(cuda)).sum(), [xg, wg])
    ggxo, ggwo = torch.autograd.grad((gxo * vx).sum() + (gwo * vw).sum(), [xo, wo])
    close(nchw(ggx), ggxo, 5e-5, "double bwd wrt x")
    close(ggw, ggwo, 5e-5, "double bwd wrt w")


def test_conv_adjoint_identity_full_size(cuda, fp32_mode):
    """Size-independent property at the north-star layer's shape (B=4 to bound memory): <conv(x), y> == <x, conv^T(y)>."""
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(4, 256, 256, 128, device=cuda, generator=g)
    yv = torch.randn(4, 256, 256, 128, device=cuda, generator=g)
    w = torch.randn(9, 128, 128, device=cuda, generator=g) / math.sqrt(1152)
    lhs = (ops.conv2d(x, w, 3, 0) * yv).double().sum()
    rhs = (x * ops.conv2d(yv, w, 3, 0, flip=True, transposed=True)).double().sum()
    assert abs(lhs - rhs) / abs(lhs) < 1e-5


# ------------------------------------------------------------------------------------------------ modulated conv
@pytest.mark.parametrize("tag,ci,co,k,demod,up,hw", [("plain", 32, 16, 3, True, False, 8), ("up", 16, 32, 3, True, True, 5),
                                                      ("rgb", 32, 3, 1, False, False, 8)])
def test_modulated_conv_golden(cuda, fp32_mode, tag, ci, co, k, demod, up, hw):
    from gif_b200.model import stylegan2_common_layers as cl
    g = gu.load_golden("modconv.npz")
    m = cl.ModulatedConv2d(ci, co, k, 512, demodulate=demod, upsample=up).to(cuda)
    m.weight.data = gu.randn((1, co, ci, k, k), 20).to(cuda)
    m.modulation.weight.data = gu.randn((ci, 512), 21).to(cuda)
    m.modulation.bias.data = (1.0 + 0.1 * gu.randn((ci,), 22)).to(cuda)
    x = gu.randn((3, ci, hw, hw), 23).to(cuda).requires_grad_(True)
    st = gu.randn((3, 512), 24).to(cuda).requires_grad_(True)
    y = m(x, st)
    close(y, g[f"{tag}_y"], 5e-5, "y")
    gy = gu.randn(tuple(y.shape), 25).to(cuda)
    grads = torch.autograd.grad((y * gy).sum(), [x, st, m.weight, m.modulation.weight, m.modulation.bias])
    for n, gr in zip("x style w modw modb".split(), grads):
        close(gr, g[f"{tag}_g{n}"], 1e-4, f"grad {n}")


def test_modulated_conv_config1(cuda, fp32_mode):
    """BASELINE.json configs[0]: ModulatedConv2d(512,512,3,512), x (4,512,64,64) -- sampled golden of the reference."""
    from gif_b200.model import stylegan2_common_layers as cl
    g = gu.load_golden("modconv.npz")
    m = cl.ModulatedConv2d(512, 512, 3, 512).to(cuda)
    m.weight.data = gu.randn((1, 512, 512, 3, 3), 30).to(cuda)
    m.modulation.weight.data = gu.randn((512, 512), 31).to(cuda)
    with torch.no_grad():
        y = m(gu.randn((4, 512, 64, 64), 32).to(cuda), gu.randn((4, 512), 33).to(cuda))
    s, tot = gu.sample(y, 4096, 1)
    e = np.abs(s - g["config1_sample"]).max() / float(g["config1_absmax"])
    assert e < 5e-5, e
    assert abs(tot - float(g["config1_sum"])) / (float(g["config1_absmax"]) * math.sqrt(y.numel())) < 1e-4


@pytest.mark.parametrize("m,n,k,ta,tb", [(32, 512, 8192, False, True), (512, 8192, 32, True, False), (32, 8192, 512, False, False),
                                         (3, 16, 24, False, True), (70, 33, 1500, False, True)])
def test_sgemm_shapes_incl_split_k(cuda, m, n, k, ta, tb):
    """EqualLinear GEMMs incl. the split-K path (8192 -> 512 discriminator head) and ragged edges, fwd + both gradients."""
    from gif_b200 import ops
    a = gu.randn((k, m) if ta else (m, k), 1)
    b = gu.randn((n, k) if tb else (k, n), 2)
    ag, bg = a.to(cuda).requires_grad_(True), b.to(cuda).requires_grad_(True)
    c = ops.matmul(ag, bg, ta, tb, alpha=0.5)
    ao, bo = a.double().requires_grad_(True), b.double().requires_grad_(True)
    co = 0.5 * (ao.t() if ta else ao) @ (bo.t() if tb else bo)
    close(c, co, 2e-5, "C")
    g = gu.randn((m, n), 3)
    ga, gb = torch.autograd.grad(c, [ag, bg], g.to(cuda))
    gao, gbo = torch.autograd.grad(co, [ao, bo], g.double())
    close(ga, gao, 2e-5, "dA")
    close(gb, gbo, 2e-5, "dB")


# ------------------------------------------------------------------------------------------------ fused first-order backwards
@pytest.mark.parametrize("c", [32, 64, 128, 96, 20])
def test_fused_tail_and_scale_backward(cuda, fp32_mode, c):
    """first-order backward (no create_graph) of the StyledConv tail and of the input modulation: the single-pass
    kernels (16-byte variants for C % 32 == 0 with 8/16/32 channel lanes, scalar otherwise) against torch autograd on the
    same formulas, and against this package's own closed-set (create_graph=True) path."""
    from gif_b200 import ops
    b, h, w = 3, 13, 11
    acc = gu.randn((b, h, w, c), 31).to(cuda)
    d = (gu.rand_uniform((b, c), 32) + 1.5).to(cuda)
    noise = gu.randn((b, h, w, c), 33).to(cuda)
    bias = gu.randn((c,), 34).to(cuda)
    gy = gu.randn((b, h, w, c), 35).to(cuda)
    s = gu.randn((b, c), 36).to(cuda)

    def ours(create_graph):
        a, dd, nn, bb, ss = (t.clone().requires_grad_(True) for t in (acc, d, noise, bias, s))
        y = ops.bias_act(ops.chan_scale(a, ss), bb, 0.2, math.sqrt(2.0), rowscale=dd, add=nn)
        return torch.autograd.grad(y, (a, dd, nn, bb, ss), gy, create_graph=create_graph)

    a, dd, nn, bb, ss = (t.clone().requires_grad_(True) for t in (acc, d, noise, bias, s))
    pre = (a * ss[:, None, None, :]) * dd[:, None, None, :] + nn + bb
    ref = torch.autograd.grad(torch.nn.functional.leaky_relu(pre, 0.2) * math.sqrt(2.0), (a, dd, nn, bb, ss), gy)
    for name, g1, g2, r in zip(("acc", "demod", "noise", "bias", "style"), ours(False), ours(True), ref):
        close(g1, r, TOL32, f"fused first-order grad[{name}]")
        close(g2, r, TOL32, f"closed-set grad[{name}]")


def test_cross_block_reductions_are_bitwise_reproducible(cuda, fp32_mode):
    """The gradient reductions over pixels (bias / demodulation / style gradients, ToRGB weights, split-K GEMMs) add their
    per-block partial sums in a fixed order: repeated calls give the same bits, so a training run is reproducible."""
    from gif_b200 import ops
    b, h, w, c = 4, 96, 96, 128
    acc, noise, gy = (gu.randn((b, h, w, c), s).to(cuda) for s in (41, 42, 43))
    d, s = (gu.rand_uniform((b, c), 44) + 1.5).to(cuda), gu.randn((b, c), 45).to(cuda)
    bias = gu.randn((c,), 46).to(cuda)
    wrgb = gu.randn((3, c), 47).to(cuda)
    ga, gb = gu.randn((32, 8192), 48).to(cuda), gu.randn((512, 8192), 49).to(cuda)

    def grads():
        a, dd, bb, ss, ww = (t.clone().requires_grad_(True) for t in (acc, d, bias, s, wrgb))
        y = ops.bias_act(ops.chan_scale(a, ss), bb, 0.2, math.sqrt(2.0), rowscale=dd, add=noise)
        out = list(torch.autograd.grad(y, (dd, bb, ss), gy))
        out.append(ops.rows_sum(gy.reshape(b, h * w, c)))
        x, m = ga.clone().requires_grad_(True), gb.clone().requires_grad_(True)
        y = ops.matmul(x, m, False, True)            # 16 output tiles, K = 8192: the split-K path
        out.append(y.detach())
        out += torch.autograd.grad(y, (x, m), gu.randn((32, 512), 50).to(cuda))
        return out
    first = grads()
    for _ in range(3):
        for g0, g1 in zip(first, grads()):
            assert torch.equal(g0, g1)


@pytest.mark.parametrize("c", [32, 64, 128, 20])
def test_fused_second_order_tail_and_scale(cuda, fp32_mode, c):
    """The create_graph backward taken inside ``ops.input_gradient_only()`` (path-length regulariser): one node per tail /
    modulation with the fused second-order kernel gifb200_tail_bwd2, against torch's own double backward of the same
    formulas and against this package's closed-set composition (16-byte and scalar kernel variants)."""
    import contextlib
    from gif_b200 import ops
    b, h, w = 3, 13, 11
    acc = gu.randn((b, h, w, c), 41).to(cuda)
    d = (gu.rand_uniform((b, c), 42) + 1.5).to(cuda)
    noise = gu.randn((b, h, w, c), 43).to(cuda)
    bias = gu.randn((c,), 44).to(cuda)
    gy = gu.randn((b, h, w, c), 45).to(cuda)
    r = gu.randn((b, h, w, c), 46).to(cuda)
    rd = gu.randn((b, c), 47).to(cuda)
    names = ("gacc", "gd", "d2/dgy", "d2/dacc", "d2/dd")

    def tail(fused, torch_ref=False):
        a, dd, g = (t.clone().requires_grad_(True) for t in (acc, d, gy))
        if torch_ref:
            y = torch.nn.functional.leaky_relu(a * dd[:, None, None, :] + noise + bias, 0.2) * math.sqrt(2.0)
        else:
            y = ops.bias_act(a, bias, 0.2, math.sqrt(2.0), rowscale=dd, add=noise)
        with (ops.input_gradient_only() if fused else contextlib.nullcontext()):
            ga, gd = torch.autograd.grad(y, (a, dd), g, create_graph=True)
        return (ga, gd) + torch.autograd.grad((ga * r).sum() + (gd * rd).sum(), (g, a, dd))

    ref = tail(False, torch_ref=True)
    for name, g1, g2, rr in zip(names, tail(True), tail(False), ref):
        close(g1, rr, TOL32, f"fused second-order tail {name}")
        close(g2, rr, TOL32, f"closed-set second-order tail {name}")
    # one upstream gradient only (the other output unused): the NULL branches of the kernel
    for use in (0, 1):
        outs = []
        for fused in (True, False):
            a, dd, g = (t.clone().requires_grad_(True) for t in (acc, d, gy))
            y = ops.bias_act(a, bias, 0.2, math.sqrt(2.0), rowscale=dd, add=noise)
            with (ops.input_gradient_only() if fused else contextlib.nullcontext()):
                first = torch.autograd.grad(y, (a, dd), g, create_graph=True)
            L = (first[0] * r).sum() if use == 0 else (first[1] * rd).sum()
            outs.append(torch.autograd.grad(L, (g, a, dd), allow_unused=True))
        for name, g1, g2 in zip(names[2:], *outs):
            assert (g1 is None) == (g2 is None) or (g1 is None and float(g2.abs().max()) == 0.0), name
            if g1 is not None and g2 is not None:
                close(g1, g2, TOL32, f"fused second-order tail, upstream {use}: {name}")

    # the modulation variant (no mask): gx = gxs*s, gs = sum gxs*x
    s = gu.randn((b, c), 48).to(cuda)
    gxs0 = gu.randn((b, h, w, c), 49).to(cuda)

    def scale(fused):
        g, x, ss = (t.clone().requires_grad_(True) for t in (gxs0, acc, s))
        if fused:
            gx, gs = ops._TailBwdCG.apply(g, None, x, ss, 1.0, 1.0, False)
        else:
            gx, gs = g * ss[:, None, None, :], (g * x).sum((1, 2))
        return (gx, gs) + torch.autograd.grad((gx * r).sum() + (gs * rd).sum(), (g, x, ss))

    for name, g1, rr in zip(("gx", "gs", "d2/dgxs", "d2/dx", "d2/ds"), scale(True), scale(False)):
        close(g1, rr, TOL32, f"fused second-order modulation {name}")


@pytest.mark.parametrize("c", [32, 64, 128, 512, 20])
def test_torgb_kernels(cuda, fp32_mode, c):
    """ToRGB contraction y[b,p,k] = sum_i x[b,p,i] ws[b,k,i]: the 16-byte kernels (8 / 16 / 32 channel lanes, several
    channel chunks per lane at C = 512, ragged pixel counts) and the scalar fallback; forward, both gradients, and the
    second derivative closure, against torch einsum."""
    from gif_b200 import ops
    b, h, w = 3, 7, 9
    x = gu.randn((b, h, w, c), 41).to(cuda).requires_grad_(True)
    ws = gu.randn((b, 3, c), 42).to(cuda).requires_grad_(True)
    gy = gu.randn((b, h, w, 3), 43).to(cuda)
    y = ops.torgb(x, ws)
    xr, wr = x.detach().clone().requires_grad_(True), ws.detach().clone().requires_grad_(True)
    yr = torch.einsum("bhwi,bki->bhwk", xr, wr)
    close(y, yr, TOL32, "torgb fwd")
    gx, gw = torch.autograd.grad(y, (x, ws), gy, create_graph=True)
    gxr, gwr = torch.autograd.grad(yr, (xr, wr), gy, create_graph=True)
    close(gx, gxr, TOL32, "torgb grad x")
    close(gw, gwr, TOL32, "torgb grad ws")
    v = gu.randn((b, h, w, c), 44).to(cuda)
    (g2,) = torch.autograd.grad((gx * v).sum(), ws)
    (g2r,) = torch.autograd.grad((gxr * v).sum(), wr)
    close(g2, g2r, TOL32, "torgb second derivative")
