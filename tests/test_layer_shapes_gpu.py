"""The persistent convolution and FIR kernels at the 256^2 training step's layer shapes, against float64.

conv_tc_kernel, wgrad_tc_kernel and the pipelined FIR kernels (upfirdn2d_fir4_pipe_kernel<1/2>, upfirdn2d_up2_pipe_kernel)
are persistent: a CTA walks a list of tiles and keeps its shared-memory ring, mbarrier phase bits or cp.async double buffer
running from one tile to the next.  What only runs at real sizes -- a CTA's second and later tiles, the buffer that flips
between tiles, a main loop that wraps the stage ring dozens of times, a ragged last round -- is what each case here is for.

Every case is a row with the mechanism it exists for.  The CPU test restates the small launch arithmetic of the host code
(tile edge, grid cap, tile count, k-steps) and asserts that each case reaches its mechanism: at least three tiles per CTA
(two rounds past the first, so a double buffer is refilled and read again) with a ragged last round, and that the batch is
the smallest that does.  The GPU tests confirm the same facts through the library: the tile from the profiled kernel name,
no split-K from gifb200_conv2d_workspace_bytes being only the staged weights, the weight-gradient path and its split count
from gifb200_conv2d_wgrad_path / _workspace_bytes.

References are float64 torch (test_second_order_tc_gpu.ref_conv, oracle.stylegan2_oracle.upfirdn2d).  Bars: 2e-5 in tf32
on tf32-rounded inputs, 5e-5 in bf16x3 on raw inputs, max-norm and L2; 1e-5 for the fp32 FIR (16 products per output).

Weight gradients get one more term.  The tensor cores' fp32 accumulator does not round to nearest: the error of a register
grows linearly with the number n of MMA results added into it, as a truncating accumulator's would, by up to half an ulp per
step: n * 2^-24 relative.  Measured on an H100 80GB HBM3 (700 W) the error is about a third of that in every case here,
forward and backward, in both modes.  The forward's 144 k-steps
(576 or 864 steps) stay inside the mode's bar, but a weight-gradient CTA of a 512-channel layer sums hundreds of 32-pixel
units into one register (3200 steps at B = 25 in tf32): 6e-5 in tf32 and 9e-5 in bf16x3, where the exact-fp32 SIMT kernel on
the same inputs stays below 1e-5.  So the weight gradient is held to the mode's bar plus n * 2^-24, n from the launch plan,
and the SIMT kernel's error is printed beside it and must be inside the mode's bar."""
import math
import os

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

# Kineto tears CUPTI down at the end of every profiling window and re-initialises it at the next one.  torch.profiler
# turns that teardown off itself when CUDA graphs are in use: re-initialisation after a graph capture is unreliable.  In a
# full suite run the trainer tests capture graphs (test_dropin_train_gpu.py) before the kernel-name checks here run, and
# windows opened after that re-initialisation missed every kernel record five times in a row.  So the kernel-name checks
# keep CUPTI set up for the whole test process, from before the first window opens.
os.environ.setdefault("TEARDOWN_CUPTI", "0")

import golden_util as gu
from oracle import stylegan2_oracle as O
from test_second_order_tc_gpu import S1, S2, T2, ADJ, assert_close, in_hw, out_hw, ref_conv, tensor_cores_only

SMS = 132                                   # kNumSMs (common.cuh), H100 SXM
BAR = {"tf32": 2e-5, "bf16x3": 5e-5}
FIR_BAR = 1e-5
# accumulate steps per 32-pixel unit into one weight-gradient register: 4 mma.m16n8k8 (tf32); 2 slices x 3 wgmma.k16 (bf16x3)
WGRAD_STEPS_PER_UNIT = {"tf32": 4, "bf16x3": 6}


# ------------------------------------------------------------------------------------------------ launch arithmetic
def conv_plan(B, Hi, Wi, Ci, Co, k, mode):
    """conv_tc.cu's host arithmetic for one gifb200_conv2d launch (pick_ksplit, pick_tile, tile_geometry, launch):
    CTA tile, K splits, tiles, persistent grid and k-steps (32-channel stages) per tile of each phase."""
    Ho, Wo = out_hw(Hi, Wi, k, mode)
    Hs, Ws = (Hi, Wi) if mode == T2 else (Ho, Wo)
    nphase = 4 if mode == T2 else 1

    def mtiles(bm):
        wt = min(Ws, 128)
        ht = min(bm // wt, Hs)
        nt = bm // (wt * ht)
        return (Ws // wt) * (Hs // ht) * -(-B // nt)

    bm, bn = 128, next(b for b in (128, 64, 32) if Co % b == 0)
    iters = k * k * (Ci // 32)
    ks = 1
    if mode != T2 and mtiles(128) * (Co // bn) <= SMS // 2 and iters >= 8:
        ks = min(2 * SMS // (mtiles(128) * (Co // bn)), iters // 4, 16)
        ks = ks if ks >= 2 else 1
    if ks == 1 and Co % 128 == 0:
        lbm, lbn = (128, 256) if Co % 256 == 0 else (256, 128)
        if mtiles(lbm) * (Co // lbn) * nphase >= 3 * SMS // 4:
            bm, bn = lbm, lbn
    tiles = mtiles(bm) * (Co // bn) * nphase * ks
    grid = min(tiles, (1 if bm * bn > 128 * 128 else 2) * SMS)
    taps = (4, 2, 2, 1) if mode == T2 else (k * k,)
    return dict(tile=(bm, bn), ksplit=ks, tiles=tiles, grid=grid, ksteps=tuple(t * (Ci // 32) // ks for t in taps))


def wgrad_plan(B, Hi, Wi, Ci, Co, k, mode):
    """conv_wgrad_tc.cu's split of the pixel loop for the wide variant (small channels Cs % 128 == 0): one CTA per
    (128 small channels, 64 big channels, kernel row, split), one wave; a CTA sums ``units_per_cta`` 32-pixel units."""
    Ho, Wo = out_hw(Hi, Wi, k, mode)
    Hs, Ws, Cs, Cb = (Hi, Wi, Ci, Co) if mode == T2 else (Ho, Wo, Co, Ci)
    assert Cs % 128 == 0 and Cb % 64 == 0
    units = B * Hs * Ws // 32
    splits = max(1, min(SMS // ((Cs // 128) * (Cb // 64) * k), units))
    return dict(splits=splits, units_per_cta=-(-units // splits))


def fir_plan(B, Hi, Wi, C, Ho, Wo, up, down, py0):
    """upfirdn2d.cu's choice of pipe kernel for a 4x4 FIR with C % 32 == 0, its output tile edge, tiles and grid."""
    if up == 2 and down == 1 and Ho >= 8 and Wo >= 8 and 0 <= py0 <= 3:
        name, edge, cap = "upfirdn2d_up2_pipe_kernel", 16, 4 * SMS
    elif up == 1 and down in (1, 2) and Ho >= 4 and Wo >= 4:
        name, edge, cap = f"upfirdn2d_fir4_pipe_kernel<{down}>", 16 if down == 1 else 8, 2 * SMS
    else:
        return None
    tiles = B * -(-Ho // edge) * -(-Wo // edge) * (C // 32)
    return dict(kernel=name, tiles=tiles, grid=min(tiles, cap))


def reaches(plan):
    """Two rounds past the first (every CTA runs at least three tiles) and a ragged last round."""
    return plan["tiles"] >= 3 * plan["grid"] and plan["tiles"] % plan["grid"] != 0


def fir_launches(B, H, W, C, up, down, pad):
    """Plans of the forward call and of its autograd adjoint (_UpFirDn.backward: up and down swapped, pad0' = 3 - pad0,
    flipped kernel, output = the forward's input)."""
    Ho, Wo = ((H * up + pad[0] + pad[1] - 4) // down + 1, (W * up + pad[0] + pad[1] - 4) // down + 1)
    return (fir_plan(B, H, W, C, Ho, Wo, up, down, pad[0]), fir_plan(B, Ho, Wo, C, H, W, down, up, 3 - pad[0]))


# ------------------------------------------------------------------------------------------------ the cases
# (B, Hs, Ws, Ci, Co, mode, tile, k-steps per phase, mechanism); Hs x Ws is the SITE grid (output for S1 / S2, input for
# T2), 3x3 kernels.  B is the smallest batch with which the forward launch reaches (checked below); the step runs 32.
CONV_CASES = [
    (25, 32, 32, 512, 512, S1, (128, 256), (144,), "144 k-steps per tile (the 4-stage ring wraps 36 times) on 128x256 tiles"),
    (25, 32, 32, 512, 512, S2, (128, 256), (144,), "stride-2 5-D boxes over 144 k-steps; the input gradient is a 4-phase T2"),
    (25, 16, 16, 512, 512, T2, (128, 256), (64, 32, 32, 16),
     "4 phases rotated from round to round, plus the border launches and the corner kernel at Ci = Co = 512"),
    (4, 64, 64, 512, 256, T2, (128, 256), (64, 32, 32, 16), "4 phases at Co = 256; the input gradient is an S2 with Co = 512"),
    (4, 128, 128, 256, 256, S1, (128, 256), (72,), "128x256 tiles with Ci = 256: 72 k-steps over one-row site boxes"),
    (2, 256, 256, 128, 128, S1, (256, 128), (36,), "256x128 tiles with Ci = 128; the weight gradient in 22 splits"),
]
CONV_IDS = [f"{'S1 S2 T2'.split()[c[5]]}-{c[3]}to{c[4]}-{c[1]}sq-B{c[0]}" for c in CONV_CASES]

# (B, H, W, C, up, down, pad, gain of the model's blur kernel, mechanism); B is the smallest batch with which BOTH the
# forward launch and its adjoint reach.
FIR_CASES = [
    (1, 256, 256, 128, 1, 1, (2, 2), 1.0, "D's blur before the 256^2 stride-2 conv: 257^2 output, ragged tile edge"),
    (4, 64, 64, 512, 1, 1, (2, 2), 1.0, "16 channel chunks in the tile decode"),
    (1, 257, 257, 128, 1, 1, (1, 1), 4.0, "G's blur after the 256^2 T2 conv"),
    (2, 256, 256, 128, 1, 2, (1, 1), 1.0, "D's skip (fir4<2>); its adjoint is the up2 pipe kernel with flip = 1, pad 2"),
    (7, 64, 64, 128, 2, 1, (0, 0), 4.0, "up2 pipe kernel at pad 0"),
    (7, 64, 64, 128, 2, 1, (1, 1), 4.0, "up2 pipe kernel at pad 1"),
    (5, 64, 64, 128, 2, 1, (2, 2), 4.0, "up2 pipe kernel at pad 2, ragged tile edge"),
    (5, 64, 64, 128, 2, 1, (3, 3), 4.0, "up2 pipe kernel at pad 3, ragged tile edge"),
]
FIR_IDS = [f"{'up2' if c[4] == 2 else 'down2' if c[5] == 2 else 'blur'}-pad{c[6][0]}-{c[1]}sq-C{c[3]}-B{c[0]}"
           for c in FIR_CASES]


def conv_launches(B, Hs, Ws, Ci, Co, mode):
    Hi, Wi = in_hw(Hs, Ws, mode)
    Ho, Wo = out_hw(Hi, Wi, 3, mode)
    return (conv_plan(B, Hi, Wi, Ci, Co, 3, mode), conv_plan(B, Ho, Wo, Co, Ci, 3, ADJ[mode]),
            wgrad_plan(B, Hi, Wi, Ci, Co, 3, mode))


def test_reach_cpu():
    """Each case reaches the mechanism of its row, with the smallest batch that does; printed as a table."""
    print()
    for B, Hs, Ws, Ci, Co, mode, tile, ksteps, why in CONV_CASES:
        fwd, adj, wg = conv_launches(B, Hs, Ws, Ci, Co, mode)
        print(f"  conv {'S1 S2 T2'.split()[mode]} {Ci}->{Co} site {Hs}^2 B={B}: tile {fwd['tile']}, {fwd['tiles']} tiles on "
              f"{fwd['grid']} CTAs ({fwd['tiles'] / fwd['grid']:.2f} rounds), k-steps {fwd['ksteps']}; input gradient "
              f"{adj['tile']} {adj['tiles'] / adj['grid']:.2f} rounds; wgrad {wg['splits']} splits x "
              f"{wg['units_per_cta']} units  -- {why}")
        assert fwd["ksplit"] == 1 and fwd["tile"] == tile and fwd["ksteps"] == ksteps, (why, fwd)
        assert reaches(fwd), (why, fwd)
        assert B == 1 or not reaches(conv_launches(B - 1, Hs, Ws, Ci, Co, mode)[0]), f"{why}: B = {B - 1} reaches too"
        assert adj["ksplit"] == 1, (why, adj)
    for B, H, W, C, up, down, pad, _, why in FIR_CASES:
        launches = fir_launches(B, H, W, C, up, down, pad)
        print("  fir " + ", ".join(f"{p['kernel']} {p['tiles']} tiles on {p['grid']} CTAs ({p['tiles'] / p['grid']:.2f} rounds)"
                                   for p in launches) + f"  -- {why}")
        assert all(p is not None and reaches(p) for p in launches), (why, launches)
        assert B == 1 or not all(reaches(p) for p in fir_launches(B - 1, H, W, C, up, down, pad)), f"{why}: B = {B - 1} reaches too"
    # the adjoint of the decimating FIR is the only call of the up2 pipe kernel with a flipped kernel
    assert fir_launches(*FIR_CASES[3][:7])[1]["kernel"] == "upfirdn2d_up2_pipe_kernel"
    assert {fir_launches(*c[:7])[0]["kernel"] for c in FIR_CASES} == {
        "upfirdn2d_fir4_pipe_kernel<1>", "upfirdn2d_fir4_pipe_kernel<2>", "upfirdn2d_up2_pipe_kernel"}


# ------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(params=["tf32", "bf16x3"])
def tc_precision(request):
    from gif_b200 import ops
    old = ops.get_precision()
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(old)


def kernel_names(fn, ok):
    """Names of the kernels ``fn`` launches, from torch.profiler.  With CUDA activity alone, a profiling window now and then
    delivers no kernel records at all (the window holds only an activity-buffer request); CPU activity is recorded too,
    and ``fn`` is profiled again, up to five times in all, until ``ok(names)``."""
    for _ in range(5):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.key for e in prof.key_averages()}
        if ok(names):
            break
    return names


def template_args(names, kernel):
    """The template argument lists of every profiled instantiation of ``kernel``."""
    return {n.split(kernel + "<", 1)[1].split(">", 1)[0].replace(" ", "") for n in names if kernel + "<" in n}


def staged_weight_bytes(Ci, Co, k):
    return -(-(k * k * Co * Ci * 4 + 256) // 256) * 256


# ------------------------------------------------------------------------------------------------ convolutions
@pytest.mark.gpu
@pytest.mark.parametrize("B,Hs,Ws,Ci,Co,mode,tile,ksteps,why", CONV_CASES, ids=CONV_IDS)
def test_conv_at_layer_shape(cuda, tc_precision, B, Hs, Ws, Ci, Co, mode, tile, ksteps, why):
    """Forward, input gradient (ops.conv2d autograd: the (True, True) S1 and (False, True) S2 <-> T2 adjoints) and weight
    gradient (_ConvWgrad) against float64; the launch plan through the library."""
    from gif_b200 import ops
    from gif_b200._lib import lib
    precision, k = tc_precision, 3
    impl = 3 if precision == "bf16x3" else 2
    Hi, Wi = in_hw(Hs, Ws, mode)
    Ho, Wo = out_hw(Hi, Wi, k, mode)
    fwd, adj, wg = conv_launches(B, Hs, Ws, Ci, Co, mode)
    # no split-K (the workspace is the staged weights alone) on the forward and the input-gradient launch; the wide
    # weight-gradient kernel with the restated split count
    assert lib.gifb200_conv2d_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, 0, impl) == staged_weight_bytes(Ci, Co, k)
    assert lib.gifb200_conv2d_workspace_bytes(B, Ho, Wo, Co, Hi, Wi, Ci, k, ADJ[mode], 1, impl) == staged_weight_bytes(Ci, Co, k)
    assert lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl) == impl
    assert lib.gifb200_conv2d_wgrad_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl) == \
        wg["splits"] * k * k * Co * Ci * 4 + 256

    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Hs + Ci + Co + mode)
    x = torch.randn(B, Hi, Wi, Ci, device=cuda, generator=g)
    w = torch.randn(k * k, Co, Ci, device=cuda, generator=g) / math.sqrt(k * k * Ci)
    gy = torch.randn(B, Ho, Wo, Co, device=cuda, generator=g)
    if precision == "tf32":
        x, w, gy = (ops._round_tf32_raw(t) for t in (x, w, gy))

    x3 = "true" if precision == "bf16x3" else "false"
    want = {f"{p['tile'][0]},{p['tile'][1]},{x3}" for p in (fwd, adj)}
    out = {}

    def run():
        with tensor_cores_only(precision):
            xg, wg_ = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
            out["y"] = ops.conv2d(xg, wg_, k, mode)
            out["gx"], out["gw"] = torch.autograd.grad(out["y"], (xg, wg_), gy)

    names = kernel_names(run, lambda ns: want <= template_args(ns, "conv_tc_kernel") and template_args(ns, "wgrad_tc_kernel"))
    tiles = template_args(names, "conv_tc_kernel")
    assert want <= tiles, (why, want, tiles)
    wargs = template_args(names, "wgrad_tc_kernel")
    assert wargs and all(a.split(",")[2] == "false" and a.split(",")[-1] == "4" for a in wargs), wargs   # wide, not STACK

    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yr = ref_conv(xr, wr, k, mode)
    gxr, gwr = torch.autograd.grad(yr, (xr, wr), gy.double())
    old = ops.CONV_IMPL
    ops.CONV_IMPL = 1
    try:
        gw_simt = ops._wgrad_raw(x, gy, k, mode, False, False)
    finally:
        ops.CONV_IMPL = old
    print(f"\n  {why}")
    assert_close("y", out["y"], yr, precision, bar=BAR[precision])
    assert_close("gx", out["gx"], gxr, precision, bar=BAR[precision])
    assert_close("gw simt fp32", gw_simt, gwr, "fp32", lower=False, bar=BAR[precision])
    steps = wg["units_per_cta"] * WGRAD_STEPS_PER_UNIT[precision]
    print(f"  gw: {wg['units_per_cta']} units = {steps} accumulate steps per register: bar {BAR[precision]:.0e} + "
          f"{steps} x 2^-24")
    assert_close("gw", out["gw"], gwr, precision, bar=BAR[precision] + steps * 2.0 ** -24)


# ------------------------------------------------------------------------------------------------ FIR
def fir_kernel(kind, gain):
    """The model's blur kernel (outer([1,3,3,1]) / 64 * gain: separable), or a random 4x4 one that is neither separable
    nor symmetric under the flip of the adjoint."""
    if kind == "blur":
        return gu.blur_kernel(gain)
    k = torch.randn(4, 4, generator=torch.Generator().manual_seed(17)) / 4.0
    assert not torch.allclose(k, k.flip(0, 1))
    return k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["blur", "random"])
@pytest.mark.parametrize("B,H,W,C,up,down,pad,gain,why", FIR_CASES, ids=FIR_IDS)
def test_fir_at_layer_shape(cuda, fp32_mode, B, H, W, C, up, down, pad, gain, why, kind):
    """Forward and autograd adjoint in fp32 against float64; the pipe kernel of both calls from the profile."""
    from gif_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 100 + H + C + up * 10 + down + pad[0])
    kern = fir_kernel(kind, gain).to(cuda)
    x = torch.randn(B, H, W, C, device=cuda, generator=g)
    Ho, Wo = (ops.upfirdn_out_size(n, 4, up, down, pad[0], pad[1]) for n in (H, W))
    gy = torch.randn(B, Ho, Wo, C, device=cuda, generator=g)
    plans = fir_launches(B, H, W, C, up, down, pad)
    out = {}

    def run():
        xg = x.clone().requires_grad_(True)
        out["y"] = ops.upfirdn2d(xg, kern, up, down, pad)
        (out["gx"],) = torch.autograd.grad(out["y"], xg, gy)

    names = kernel_names(run, lambda ns: all(any(p["kernel"] in n for n in ns) for p in plans))
    for plan in plans:
        assert any(plan["kernel"] in n for n in names), (why, plan["kernel"], [n for n in names if "upfirdn" in n])
    y, gx = out["y"], out["gx"]

    xr = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    yr = O.upfirdn2d(xr, kern.double(), up, down, pad)
    (gxr,) = torch.autograd.grad(yr, xr, gy.double().permute(0, 3, 1, 2))
    print(f"\n  {why} [{kind}]")
    assert_close("y", y, yr.permute(0, 2, 3, 1), "fp32", lower=False, bar=FIR_BAR)
    assert_close("gx", gx, gxr.permute(0, 2, 3, 1), "fp32", lower=False, bar=FIR_BAR)


@pytest.mark.gpu
def test_fir_round_tf32_at_layer_shape(cuda, fp32_mode):
    """rt=True (a tf32 convolution consumes the output): every value is round_tf32 of the fp32 result -- tf32-representable,
    within 2^-11 of it, and equal to the library's own rounding of it."""
    from gif_b200 import ops
    B, H, W, C, up, down, pad, gain, _ = FIR_CASES[0]
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(B, H, W, C, device=cuda, generator=g)
    kern = gu.blur_kernel(gain).to(cuda)
    y = ops.upfirdn2d(x, kern, up, down, pad)
    yt = ops.upfirdn2d(x, kern, up, down, pad, rt=True)
    assert int((yt.view(torch.int32) & 0x1FFF).count_nonzero()) == 0
    assert bool(((yt - y).abs() <= 2.0 ** -11 * y.abs()).all())
    assert torch.equal(yt, ops._round_tf32_raw(y))
    assert_close("y rt", yt, O.upfirdn2d(x.double().permute(0, 3, 1, 2), kern.double(), up, down, pad).permute(0, 2, 3, 1),
                 "fp32", lower=False, bar=2.0 ** -11)
