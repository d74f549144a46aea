"""The second-order passes of R1 and of the path-length regulariser, operator by operator, in fp32, tf32 and bf16x3,
against float64 torch references.

The training step differentiates its own backward twice: R1 (d scores / d image inside ``ops.input_gradient_only()``,
then the weight gradient of its square norm) and the path-length term (d image / d w, then its gradient).  Those passes
run branches of gif_b200.ops that no first-order test reaches: the grad-enabled backwards of _Conv (with and without its
fused epilogue), _ConvWgrad and _ModConvX3, the fused second-order node _TailBwdCG with its bf16x3 planes, _ActBwd /
spatial_dot / chan_scale as differentiable nodes, and weight gradients of input-gradient convolutions, (flip, transposed)
= (True, True) for S1 and (False, True) for T2 / S2.

References: float64 torch with the physical weight mapping of gifb200.h, and the leaky-ReLU masks taken from the CUDA
forward output, m = where(y > 0, 1, slope) * gain (what act_bwd / tail_bwd use).  Every reference is then linear in the
tensors a mask depends on, so the bars are operator bars, checked in max-norm (golden_util.rel_err) and in L2:
5e-5 in fp32, 1e-4 in bf16x3 (two chained contractions of 5e-5 each), 2e-3 in tf32.  In the tensor-core modes the error
must also exceed 1e-8 (the exact-fp32 SIMT kernels did not run instead), and a profile shows no SIMT convolution or
weight-gradient kernel.

The slot reductions (pixel sums written as per-chunk partial sums, then added in a fixed order) are checked against float64
at production sizes, where the row chunks are ragged, at 2e-5 of max|ref|.

The float64 helpers are themselves checked on the CPU, against the definitions of gifb200.h and torch autograd."""
import contextlib
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu
from oracle import stylegan2_oracle as O

S1, S2, T2 = 0, 1, 2                        # gif_b200.ops conv modes
ADJ = {S1: S1, S2: T2, T2: S2}
SQRT2 = math.sqrt(2.0)
BAR = {"fp32": 5e-5, "bf16x3": 1e-4, "tf32": 2e-3}
FLIPS = [(False, False), (True, True), (False, True), (True, False)]


# ------------------------------------------------------------------------------------------------ float64 references
def logical_taps(w, flip, transposed):
    """W[t][o][i] (T, Co, Ci) of a physical weight buffer (gifb200.h): transposed ? w[tt][i][o] : w[tt][o][i] with
    tt = flip ? T-1-t : t."""
    W = w.transpose(1, 2) if transposed else w
    return W.flip(0) if flip else W


def ref_conv(x, w, k, mode, flip=False, transposed=False):
    """gifb200_conv2d on NHWC tensors of any dtype (float64 here)."""
    W = logical_taps(w, flip, transposed)
    co, ci = W.shape[1:]
    Wc = W.reshape(k, k, co, ci).permute(2, 3, 0, 1)
    xc = x.permute(0, 3, 1, 2)
    if mode == S1:
        y = F.conv2d(xc, Wc, padding=k // 2)
    elif mode == S2:
        y = F.conv2d(xc, Wc, stride=2)
    else:
        y = F.conv_transpose2d(xc, Wc.transpose(0, 1), stride=2)
    return y.permute(0, 2, 3, 1)


def adjoint(mode, flip, transposed):
    """(mode, flip, transposed) of the input-gradient convolution (gifb200.h)."""
    return ADJ[mode], (not flip) if mode == S1 else flip, not transposed


def lrelu_mask(y, slope, gain):
    """The activation derivative the kernels apply, from the forward OUTPUT: gain * (y > 0 ? 1 : slope), as float64."""
    return torch.full(y.shape, float(slope), dtype=torch.float64, device=y.device).masked_fill_(y > 0, 1.0) * gain


def ref_conv_bias_act(x, w, bias, k, mode, m):
    return m * (ref_conv(x, w, k, mode) + bias)


def ref_styled_conv(x, st, A, bmod, w, bias, noise, k, mode, m, eps=1e-8):
    """StyledConv with the modulation s = st A^T + bmod: demod, modulated conv, bias_act(acc, bias, rowscale=d, add=noise)."""
    s = st @ A.t() + bmod
    d = torch.rsqrt((s * s) @ (w * w).sum(0).t() + eps)
    acc = ref_conv(x * s[:, None, None, :], w, k, mode)
    return m * (acc * d[:, None, None, :] + noise + bias)


def out_hw(h, w, k, mode):
    if mode == S1:
        return h, w
    if mode == S2:
        return (h - k) // 2 + 1, (w - k) // 2 + 1
    return 2 * (h - 1) + k, 2 * (w - 1) + k


def in_hw(hs, ws, mode):
    """Input grid of a convolution whose SITE grid (output for S1 / S2, input for T2) is hs x ws."""
    return (2 * hs + 1, 2 * ws + 1) if mode == S2 else (hs, ws)


# ------------------------------------------------------------------------------------------------ CPU: the references
def direct_conv(x, w, k, mode, flip, transposed):
    """gifb200.h's definition of gifb200_conv2d, one output pixel and one tap at a time."""
    B, Hi, Wi, _ = x.shape
    T = k * k
    co = w.shape[2] if transposed else w.shape[1]
    Ho, Wo = out_hw(Hi, Wi, k, mode)
    y = x.new_zeros(B, Ho, Wo, co)
    for t in range(T):
        kh, kw = divmod(t, k)
        tt = T - 1 - t if flip else t
        Wt = w[tt].t() if transposed else w[tt]                    # (Co, Ci)
        for Y in range(Ho):
            for X in range(Wo):
                if mode == S1:
                    yi, xi = Y + kh - k // 2, X + kw - k // 2
                elif mode == S2:
                    yi, xi = 2 * Y + kh, 2 * X + kw
                elif (Y - kh) % 2 or (X - kw) % 2:
                    continue
                else:
                    yi, xi = (Y - kh) // 2, (X - kw) // 2
                if 0 <= yi < Hi and 0 <= xi < Wi:
                    y[:, Y, X] += x[:, yi, xi] @ Wt.t()
    return y


def same(a, b):
    """Equal up to float64 reassociation."""
    return float((a - b).detach().abs().max()) <= 1e-12 * float(b.detach().abs().max())


def test_float64_references_cpu():
    """ref_conv against gifb200.h's definition for every mode, k and (flip, transposed); its autograd input gradient
    against the adjoint convolution of the ABI; the pinned-mask references against torch's leaky_relu to second order."""
    g = torch.Generator().manual_seed(0)
    for k, mode in ((1, S1), (3, S1), (3, S2), (3, T2)):
        for flip, transposed in FLIPS:
            x = torch.randn(2, 5, 7, 3, generator=g, dtype=torch.float64, requires_grad=True)
            w = torch.randn(k * k, *((3, 4) if transposed else (4, 3)), generator=g, dtype=torch.float64)
            y = ref_conv(x, w, k, mode, flip, transposed)
            assert same(y, direct_conv(x.detach(), w, k, mode, flip, transposed))
            gy = torch.randn(y.shape, generator=g, dtype=torch.float64)
            (gx,) = torch.autograd.grad(y, x, gy)
            assert same(gx, ref_conv(gy, w, k, *adjoint(mode, flip, transposed)))

    # pinned masks: same first and second derivatives as autograd through leaky_relu (no pre-activation at 0 here)
    for slope, gain in ((0.2, SQRT2), (0.0, 1.0)):
        x, w, b = (torch.randn(s, generator=g, dtype=torch.float64) for s in ((2, 9, 9, 4), (9, 6, 4), (6,)))
        r = torch.randn(2, 4, 4, 6, generator=g, dtype=torch.float64)
        m = lrelu_mask(F.leaky_relu(ref_conv(x, w, 3, S2) + b, slope) * gain, slope, gain)
        outs = []
        for pinned in (True, False):
            xg, wg, bg = (t.clone().requires_grad_(True) for t in (x, w, b))
            y = ref_conv_bias_act(xg, wg, bg, 3, S2, m) if pinned else F.leaky_relu(ref_conv(xg, wg, 3, S2) + bg, slope) * gain
            (gx,) = torch.autograd.grad((y * r).sum() + 0.5 * (y * y).sum(), xg, create_graph=True)
            outs.append([gx] + list(torch.autograd.grad((gx * gx).sum(), (xg, wg, bg))))
        for a, b_ in zip(*outs):
            assert same(a, b_)

    B, Ci, Co, L = 2, 4, 5, 3
    x, st, A, bmod = (torch.randn(s, generator=g, dtype=torch.float64) for s in ((B, 4, 4, Ci), (B, L), (Ci, L), (Ci,)))
    w, bias, noise, r = (torch.randn(s, generator=g, dtype=torch.float64) for s in ((9, Co, Ci), (Co,), (B, 9, 9, Co), (B, 9, 9, Co)))
    outs = []
    for pinned in (True, False):
        xg, sg, Ag, wg = (t.clone().requires_grad_(True) for t in (x, st, A, w))
        if pinned:
            with torch.no_grad():
                pre = ref_styled_conv(x, st, A, bmod, w, bias, noise, 3, T2, 1.0)
            y = ref_styled_conv(xg, sg, Ag, bmod, wg, bias, noise, 3, T2, lrelu_mask(F.leaky_relu(pre, 0.2), 0.2, SQRT2))
        else:
            y = F.leaky_relu(ref_styled_conv(xg, sg, Ag, bmod, wg, bias, noise, 3, T2, 1.0), 0.2) * SQRT2
        (gs,) = torch.autograd.grad((y * r).sum(), sg, create_graph=True)
        outs.append([gs] + list(torch.autograd.grad((gs * gs).sum(), (xg, sg, Ag, wg))))
    for a, b_ in zip(*outs):
        assert same(a, b_)


# ------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(params=["fp32", "tf32", "bf16x3"])
def precision(request):
    from gif_b200 import ops
    old = ops.get_precision()
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(old)


@contextlib.contextmanager
def tensor_cores_only(precision):
    """In the tensor-core modes: every gifb200_conv2d and gifb200_conv2d_wgrad call made in the block takes the tensor-core
    path, by the library's own path queries on the arguments of each call (B, Hi, Wi, Ci, Ho, Wo, Co, k, mode at
    positions 3-11, transposed at 13, impl at 14 of both entry points)."""
    if precision == "fp32":
        yield
        return
    from gif_b200._lib import lib
    calls = {"gifb200_conv2d": [], "gifb200_conv2d_wgrad": []}
    originals = {name: getattr(lib, name) for name in calls}

    def spy(name):
        def call(*args):
            calls[name].append(args[3:15])
            return originals[name](*args)
        return call

    for name in calls:
        setattr(lib, name, spy(name))
    try:
        yield
    finally:
        for name, fn in originals.items():
            setattr(lib, name, fn)
    convs, wgrads = calls["gifb200_conv2d"], calls["gifb200_conv2d_wgrad"]
    assert convs and wgrads, (len(convs), len(wgrads))
    for a in convs:
        impl = a[11] & 0xF
        assert impl != 1 and lib.gifb200_conv2d_workspace_bytes(*a[:9], a[10], impl) > 0, f"SIMT convolution {a}"
    for a in wgrads:
        assert a[11] != 1 and lib.gifb200_conv2d_wgrad_path(*a[:9], a[11]) in (2, 3), f"SIMT weight gradient {a}"


def assert_close(what, got, ref, precision, lower=True, bar=None):
    """Max-norm and L2 relative error under ``bar`` (default: the mode's); above 1e-8 in the tensor-core modes when
    ``lower``."""
    assert got is not None, f"{what}: no gradient"
    a = got.detach().double().cpu().numpy()
    b = ref.detach().double().cpu().numpy()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    e_max = gu.rel_err(a, b)
    e_l2 = float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))
    bar = BAR[precision] if bar is None else bar
    print(f"  {what:<14s} [{precision:>6s}] max {e_max:.2e}  L2 {e_l2:.2e}  (bar {bar:.0e})")
    assert e_max < bar and e_l2 < bar, f"{what} [{precision}]: max {e_max:.3e}, L2 {e_l2:.3e} vs {bar:.0e}"
    if lower and precision != "fp32":
        assert e_max > 1e-8, f"{what} [{precision}]: error {e_max:.3e}: the exact-fp32 kernels ran"


def randn(g, *shape, scale=1.0):
    return torch.randn(*shape, device="cuda", generator=g) * scale


# ------------------------------------------------------------------------------------------------ conv double backward
# (B, Hs, Ws, Ci, Co, k, mode), Hs x Ws the SITE grid.  Every contraction of the recorded graph runs on the tensor cores;
# the weight gradients in it are of the forward convolution (small channels Cs = Co for S1 / S2, Ci for T2) and of the
# input-gradient convolution (Cs = Ci for S1, the low-resolution side for S2 / T2).
CONV_CASES = [
    (2, 8, 8, 128, 128, 3, S1),      # Cs = 128 both ways, narrow images (Ws < 32: multi-row boxes)
    (1, 32, 32, 64, 128, 3, S1),     # Cs = 128 / NARROW (Cs = 64), HALO (Ws >= 32)
    (2, 32, 32, 32, 64, 3, S1),      # NARROW / STACK (Cs = 32), HALO
    (2, 8, 16, 32, 32, 3, S1),       # STACK both ways, narrow images
    (2, 16, 16, 64, 32, 1, S1),      # 1x1: NARROW with Cs = 32 and Cs = 64
    (2, 8, 8, 128, 128, 1, S1),      # 1x1: Cs = 128
    (2, 8, 8, 32, 128, 3, S2),       # Cs = 128
    (1, 32, 32, 64, 64, 3, S2),      # NARROW
    (2, 8, 8, 128, 32, 3, T2),       # Cs = 128
    (1, 16, 16, 64, 64, 3, T2),      # NARROW
]


@pytest.mark.gpu
@pytest.mark.parametrize("flip,transposed", FLIPS)
@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,k,mode", CONV_CASES)
def test_conv_double_backward(cuda, precision, B, Hs, Ws, Ci, Co, k, mode, flip, transposed):
    """_Conv: gx, gw = grad(y, [x, w], gy, create_graph) then grad(<gx,vx> + <gw,vw>, [x, w, gy]); _ConvWgrad on its own:
    grad(<wgrad(x, gy), vw>, [x, gy])."""
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Hs * 10 + Ci + Co + k + mode)
    Hi, Wi = in_hw(Hs, Ws, mode)
    Ho, Wo = out_hw(Hi, Wi, k, mode)
    x = randn(g, B, Hi, Wi, Ci)
    w = randn(g, k * k, *((Ci, Co) if transposed else (Co, Ci)), scale=1.0 / math.sqrt(Ci * k * k))
    gy, vx, vw = randn(g, B, Ho, Wo, Co), randn(g, B, Hi, Wi, Ci), randn(g, *w.shape)

    with tensor_cores_only(precision):
        xg, wg, gyg = (t.clone().requires_grad_(True) for t in (x, w, gy))
        y = ops.conv2d(xg, wg, k, mode, flip, transposed)
        gx, gw = torch.autograd.grad(y, (xg, wg), gyg, create_graph=True)
        ours = [y, gx, gw] + list(torch.autograd.grad((gx * vx).sum() + (gw * vw).sum(), (xg, wg, gyg)))
        xg, gyg = (t.clone().requires_grad_(True) for t in (x, gy))
        gw1 = ops._ConvWgrad.apply(xg, gyg, k, mode, flip, transposed)
        ours += [gw1] + list(torch.autograd.grad((gw1 * vw).sum(), (xg, gyg)))

    xr, wr, gyr = (t.double().requires_grad_(True) for t in (x, w, gy))
    yr = ref_conv(xr, wr, k, mode, flip, transposed)
    gxr, gwr = torch.autograd.grad(yr, (xr, wr), gyr, create_graph=True)
    ref = [yr, gxr, gwr] + list(torch.autograd.grad((gxr * vx.double()).sum() + (gwr * vw.double()).sum(), (xr, wr, gyr),
                                                    retain_graph=True))
    ref += [gwr] + list(torch.autograd.grad((gwr * vw.double()).sum(), (xr, gyr)))
    names = ["y", "gx", "gw", "d2/dx", "d2/dw", "d2/dgy", "wgrad", "wgrad d/dx", "wgrad d/dgy"]
    for name, a, b in zip(names, ours, ref):
        assert_close(name, a, b, precision)


# ------------------------------------------------------------------------------------------------ R1 on conv2d_bias_act
R1_CASES = [
    (2, 32, 32, 64, 128, S1),        # outer weight gradient of the input-gradient conv: (flip, transposed) = (T, T), NARROW
    (2, 16, 16, 32, 32, S1),         # the noise convs' shape: STACK
    (2, 8, 8, 64, 128, S2),          # outer weight gradient of the input-gradient conv: T2 with (F, T)
]


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["input_gradient_only", "create_graph"])
@pytest.mark.parametrize("slope,gain", [(0.2, SQRT2), (0.0, 1.0)])
@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,mode", R1_CASES)
def test_r1_pass_of_conv_bias_act(cuda, precision, B, Hs, Ws, Ci, Co, mode, slope, gain, fused):
    """The inner pass: the input gradient with create_graph inside input_gradient_only (no weight gradient launched), or
    the input and weight gradients with a plain create_graph; then the outer gradients of sum |g|^2 and of sum <g, v> over
    the inner gradients, w.r.t. x, w and bias.  The upstream gradient r + y depends on y, as the gradient of the
    discriminator's later layers does."""
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 100 + Hs + Ci + Co + mode + int(slope * 10))
    Hi, Wi = in_hw(Hs, Ws, mode)
    x, w, bias = randn(g, B, Hi, Wi, Ci), randn(g, 9, Co, Ci, scale=1.0 / math.sqrt(9 * Ci)), randn(g, Co, scale=0.1)
    r = randn(g, B, Hs, Ws, Co)
    n_inner = 1 if fused else 2
    vs = [randn(g, B, Hi, Wi, Ci), randn(g, *w.shape)][:n_inner]

    with tensor_cores_only(precision):
        leaves = [t.clone().requires_grad_(True) for t in (x, w, bias)]
        y = ops.conv2d_bias_act(leaves[0], leaves[1], leaves[2], 3, mode, slope, gain)
        ops.PROFILE = []
        try:
            with (ops.input_gradient_only() if fused else contextlib.nullcontext()):
                gs = torch.autograd.grad((y * r).sum() + 0.5 * (y * y).sum(), leaves[:n_inner], create_graph=True)
            launched = [e[3] for e in ops.PROFILE]
        finally:
            ops.PROFILE = None
        assert ("wgrad" in launched) != fused, launched
        ours = [y] + list(gs) + list(torch.autograd.grad(sum((a * a).sum() for a in gs), leaves, retain_graph=True))
        ours += list(torch.autograd.grad(sum((a * b).sum() for a, b in zip(gs, vs)), leaves))

    m = lrelu_mask(y.detach(), slope, gain)
    lr = [t.double().requires_grad_(True) for t in (x, w, bias)]
    yr = ref_conv_bias_act(lr[0], lr[1], lr[2], 3, mode, m)
    gsr = torch.autograd.grad((yr * r.double()).sum() + 0.5 * (yr * yr).sum(), lr[:n_inner], create_graph=True)
    ref = [yr] + list(gsr) + list(torch.autograd.grad(sum((a * a).sum() for a in gsr), lr, retain_graph=True))
    ref += list(torch.autograd.grad(sum((a * b.double()).sum() for a, b in zip(gsr, vs)), lr))
    names = ["y"] + ["g d/dx", "g d/dw"][:n_inner] + ["|g|^2 d/dx", "|g|^2 d/dw", "|g|^2 d/db", "<g,v> d/dx", "<g,v> d/dw",
                                                       "<g,v> d/db"]
    for name, a, b in zip(names, ours, ref):
        assert_close(name, a, b, precision)


# ------------------------------------------------------------------------------------------------ path length on StyledConv
PPL_CASES = [
    (2, 16, 16, 64, 128, S1),        # C % 32 == 0, P = 256: the bf16x3 planes branches of _TailBwdCG
    (2, 8, 8, 64, 32, T2),           # the upsampling conv, P = 17^2: planes
    (2, 8, 8, 32, 32, S1),           # P = 64 < 256: _TailBwdCG's fp32 branch (still tensor-core convolutions)
]


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["input_gradient_only", "create_graph"])
@pytest.mark.parametrize("B,H,W,Ci,Co,mode", PPL_CASES)
def test_path_length_pass_of_styled_conv(cuda, precision, B, H, W, Ci, Co, mode, fused):
    """s = modulation(st); y = bias_act(modconv(x, s, w), bias, rowscale=demod(s, w), add=noise).  Inner pass: the gradient of
    <y, r> w.r.t. st inside input_gradient_only (the fused _TailBwdCG nodes), or w.r.t. (st, x, w) with a plain
    create_graph (_ModConvX3's closed-set branch); outer pass: the gradient of <g, v> w.r.t. x, st, w and the modulation."""
    from gif_b200 import ops
    L = 16
    g = torch.Generator(device="cuda").manual_seed(B * 10 + H + Ci + Co + mode)
    x, st = randn(g, B, H, W, Ci), randn(g, B, L)
    A, bmod = randn(g, Ci, L, scale=0.1), 1.0 + randn(g, Ci, scale=0.1)
    w, bias = randn(g, 9, Co, Ci, scale=1.0 / math.sqrt(9 * Ci)), randn(g, Co, scale=0.1)
    Ho, Wo = out_hw(H, W, 3, mode)
    noise, r = randn(g, B, Ho, Wo, Co), randn(g, B, Ho, Wo, Co)

    with tensor_cores_only(precision):
        leaves = [t.clone().requires_grad_(True) for t in (x, st, w, A)]
        xg, sg, wg, Ag = leaves
        s = ops.bias_act(ops.matmul(sg, Ag, False, True), bmod, 1.0, 1.0)
        d = ops.demod(s, (wg * wg).sum(0))
        acc = ops.modconv(xg, s, wg, 3, mode)
        if precision == "bf16x3":
            assert type(acc.grad_fn).__name__ == "_ModConvX3Backward", type(acc.grad_fn).__name__
        y = ops.bias_act(acc, bias, 0.2, SQRT2, rowscale=d, add=noise)
        inner = [sg] if fused else [sg, xg, wg]
        with (ops.input_gradient_only() if fused else contextlib.nullcontext()):
            gs = torch.autograd.grad((y * r).sum(), inner, create_graph=True)
        vs = [randn(g, *t.shape) for t in inner]
        ours = [y] + list(gs) + list(torch.autograd.grad(sum((a * b).sum() for a, b in zip(gs, vs)), leaves))

    m = lrelu_mask(y.detach(), 0.2, SQRT2)
    lr = [t.double().requires_grad_(True) for t in (x, st, w, A)]
    yr = ref_styled_conv(lr[0], lr[1], lr[3], bmod.double(), lr[2], bias.double(), noise.double(), 3, mode, m)
    inner_r = [lr[1]] if fused else [lr[1], lr[0], lr[2]]
    gsr = torch.autograd.grad((yr * r.double()).sum(), inner_r, create_graph=True)
    ref = [yr] + list(gsr) + list(torch.autograd.grad(sum((a * b.double()).sum() for a, b in zip(gsr, vs)), lr))
    names = ["y"] + ["g d/dst", "g d/dx", "g d/dw"][:len(inner)] + ["d2/dx", "d2/dst", "d2/dw", "d2/dmod"]
    for name, a, b in zip(names, ours, ref):
        assert_close(name, a, b, precision)


# ------------------------------------------------------------------------------------------------ upfirdn2d double backward
@pytest.mark.gpu
@pytest.mark.parametrize("up,down,pad,gain", [(2, 1, (2, 1), 4.0), (1, 2, (1, 1), 1.0), (1, 2, (2, 2), 1.0), (1, 1, (1, 1), 4.0)],
                         ids=["up2", "down2-pad1", "down2-pad2", "blur"])
def test_upfirdn2d_double_backward(cuda, precision, up, down, pad, gain):
    """The model's FIR filters at C = 128: forward, adjoint (create_graph) and the derivative of the adjoint w.r.t. its
    upstream gradient.  In tf32 the adjoint rounds its output to tf32 (a tensor-core convolution consumes it): within
    2^-11 of each value, inside the tf32 bar."""
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(up * 10 + down + pad[0] + pad[1])
    k = gu.blur_kernel(gain).to(cuda)
    x, v = randn(g, 2, 16, 16, 128), randn(g, 2, 16, 16, 128)
    xg = x.clone().requires_grad_(True)
    y = ops.upfirdn2d(xg, k, up, down, pad)
    gy = randn(g, *y.shape).requires_grad_(True)
    (gx,) = torch.autograd.grad(y, xg, gy, create_graph=True)
    (gg,) = torch.autograd.grad((gx * v).sum(), gy)

    xr, gyr = x.double().permute(0, 3, 1, 2).requires_grad_(True), gy.detach().double().permute(0, 3, 1, 2).requires_grad_(True)
    yr = O.upfirdn2d(xr, k.double(), up, down, pad)
    (gxr,) = torch.autograd.grad(yr, xr, gyr, create_graph=True)
    (ggr,) = torch.autograd.grad((gxr * v.double().permute(0, 3, 1, 2)).sum(), gyr)
    for name, a, b in (("y", y, yr), ("gx", gx, gxr), ("d2/dgy", gg, ggr)):
        assert_close(name, a, b.permute(0, 2, 3, 1), precision, lower=False)


# ------------------------------------------------------------------------------------------------ slot reductions
# Production sizes: rows per block is not a multiple of the row lanes (rows_split: 1986 rows at 256^2 with C = 128;
# rows_split_vec: 249 at 256^2, 35 at 96^2), and the last chunk is short.
@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,C", [(4, 256, 256, 32), (4, 256, 256, 128), (4, 256, 256, 512), (4, 96, 96, 128)])
def test_slot_reductions_at_production_sizes(cuda, B, H, W, C):
    """rows_sum, spatial_dot, scale_bwd (gs), tail_bwd and tail_bwd_planes (gb, gd), tail_bwd2 (gdd), torgb_bwd_w against
    float64 sums, at 2e-5 of max|ref|."""
    from gif_b200 import ops
    from gif_b200._lib import check, lib, ptr, stream
    P = H * W
    slope, gain = 0.2, SQRT2
    g = torch.Generator(device="cuda").manual_seed(B + H + C)
    gy, y, acc, gg = (randn(g, B, P, C) for _ in range(4))
    d, ggd = 0.5 + torch.rand(B, C, device=cuda, generator=g), randn(g, B, C)
    gy3 = randn(g, B, P, 3)
    m = lrelu_mask(y, slope, gain)
    gym = gy.double() * m
    errs = {}

    def close(name, got, ref):
        errs[name] = gu.rel_err(got.cpu().numpy(), ref.cpu().numpy())

    close("rows_sum", ops.rows_sum(gy), gy.double().sum(1))
    gy_acc = (gy.double() * acc.double()).sum(1)
    close("spatial_dot", ops.spatial_dot(gy, acc), gy_acc)
    gx, gs = torch.empty_like(gy), torch.empty(B, C, device=cuda)
    check(lib.gifb200_scale_bwd(ptr(gy), ptr(acc), ptr(d), ptr(gx), ptr(gs), B, P, C, 0, stream()), "scale_bwd")
    close("scale_bwd gs", gs, gy_acc)
    del gx
    gb_ref, gd_ref = gym.sum((0, 1)), (gym * acc.double()).sum(1)
    gt, gacc = torch.empty_like(gy), torch.empty_like(gy)
    gb, gd = torch.empty(C, device=cuda), torch.empty(B, C, device=cuda)
    check(lib.gifb200_tail_bwd(ptr(gy), ptr(y), ptr(acc), ptr(d), ptr(gt), ptr(gacc), ptr(gb), ptr(gd), B, P, C, slope, gain, 0,
                               stream()), "tail_bwd")
    close("tail_bwd gb", gb, gb_ref)
    close("tail_bwd gd", gd, gd_ref)
    del gt, gacc
    pt, pa = (torch.empty((2, B, P, C), dtype=torch.bfloat16, device=cuda) for _ in range(2))
    check(lib.gifb200_tail_bwd_planes(ptr(gy), ptr(y), ptr(acc), ptr(d), None, None, ptr(gb), ptr(gd), B, P, C, slope, gain,
                                      ptr(pt), ptr(pa), stream()), "tail_bwd_planes")
    close("tail_bwd_planes gb", gb, gb_ref)
    close("tail_bwd_planes gd", gd, gd_ref)
    del pt, pa, gym
    gdd = torch.empty(B, C, device=cuda)
    check(lib.gifb200_tail_bwd2(ptr(gg), ptr(ggd), ptr(gy), ptr(y), ptr(acc), ptr(d), None, None, ptr(gdd), B, P, C, slope,
                                gain, None, stream()), "tail_bwd2")
    close("tail_bwd2 gdd", gdd, (gg.double() * gy.double() * m).sum(1))
    close("torgb_bwd_w", ops._ToRgbBwdW.apply(gy3, acc), torch.einsum("bpk,bpi->bki", gy3.double(), acc.double()))
    print("  " + "  ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    bad = {k: e for k, e in errs.items() if not e < 2e-5}
    assert not bad, bad
