"""The persistent convolution at the layer shapes where its tiles start mid-ring, and the FIR pipe kernels at 32 and 64
channels: the condition-injection, stem and narrow layers of the 256^2, 512^2 and 1024^2 steps, against float64.

conv_tc_kernel's shared-memory ring index and mbarrier phase bits run on from one tile to the next, so a tile starts at
ring stage (k-steps of this CTA's earlier tiles) mod kStages, with the phase bit those wraps left.  The 128x256 / 256x128
tiles use 4 stages, the 128xBN tiles 3.  Every convolution of test_layer_shapes_gpu.py has k-steps per tile that are a
multiple of 4, so each of its tiles starts at stage 0 with a fresh phase.  The rows here are real layers whose tiles do
not: 9 or 1 k-steps on the 4-stage ring, T2 phases of 16/8/8/4 or 8/4/4/2 k-steps on the 3-stage ring.

The CPU test restates the host arithmetic of conv_tc.cu (pick_ksplit / pick_tile through test_layer_shapes_gpu.conv_plan,
kStages, decode_tile with rot_div and the T2 phase rotation, the it0 / it1 ranges of split-K) and walks every CTA's tile
list, recording the (stage, phase bit) at which each tile starts.  A row is labelled with what its forward launch reaches:
  * mid-ring: every CTA runs at least three tiles with a ragged last round (test_layer_shapes_gpu.reaches), and tiles
    start at every one of the 2 * kStages (stage, phase) states;
  * part-ring: the same, but tiles start at some of the states only: the k-steps per tile share a factor with the
    2 * kStages steps after which stage and phase repeat (2 k-steps on 4 stages: stages 0 and 2);
  * aligned: tiles start at stage 0 only.  The row is there for another mechanism, which it names: rounds of 2-CTA
    residency ("rounds": three tiles per CTA, ragged), or ragged split-K ranges ("split-K").
Each row's batch is the smallest with which the forward launch reaches its label and the weight gradient runs on the
tensor cores.  The convolution rows of test_layer_shapes_gpu.py and test_conv_tc_large_gpu.py are walked too and printed;
none of them reaches mid-ring.  The input-gradient launch of each row is walked and its label asserted as well.

The GPU test compares forward (with the model's fused epilogue), input gradient (ops.conv2d / ops.conv2d_bias_act
autograd) and weight gradient with float64, and confirms the launch plan through the library: the tiles from the profiled
conv_tc_kernel template arguments, the split-K choice from gifb200_conv2d_workspace_bytes, and the weight-gradient path,
split count and variant (STACK flag, halo, AC) from gifb200_conv2d_wgrad_path / _workspace_bytes and the profiled
wgrad_tc_kernel template arguments.  Inputs are random in every channel, including the ones the model zero-pads.

Bars are those of test_layer_shapes_gpu.py: 2e-5 in tf32 on rounded inputs, 5e-5 in bf16x3 on raw inputs, max-norm and
L2; the weight gradient's bar adds n * 2^-24, n the accumulate steps per register of the variant that ran.  With the
fused epilogue, the references take the leaky-ReLU mask from the CUDA output, as test_second_order_tc_gpu.py does; in
tf32 the input- and weight-gradient convolutions read the pre-activation gradient rounded to tf32 (the activation
backward writes it so), and their reference is taken from that same rounded operand.  An output rounded to tf32 in the
epilogue (rt) must equal the library's rounding of the unrounded output bit for bit."""
import math

import pytest
import torch

import test_layer_shapes_gpu as LS
from test_layer_shapes_gpu import (BAR, FIR_BAR, SMS, conv_plan, fir_launches, fir_plan, kernel_names, reaches,
                                   staged_weight_bytes, tc_precision, template_args, wgrad_plan)  # noqa: F401
from test_conv_tc_large_gpu import CASES as LARGE_CASES
from test_second_order_tc_gpu import S1, S2, T2, ADJ, assert_close, in_hw, lrelu_mask, out_hw, ref_conv, tensor_cores_only

# Accumulate steps per 32-pixel unit into one weight-gradient register (conv_wgrad_tc.cu):
#  * wide and STACK (AC = 4): tf32, one mma.m16n8k8 per 8-pixel step, 4 per unit; bf16x3, two 16-pixel slices of
#    three wgmmas each, 6;
#  * narrow (AC = 2): tf32, the same 4 mma.m16n8k8 per unit; bf16x3, warpgroup wg takes only slice wg of each stage, 3
#    wgmmas per unit (the two warpgroups' sums are added once at the end).
WGRAD_STEPS_PER_UNIT = {"wide": {"tf32": 4, "bf16x3": 6}, "STACK": {"tf32": 4, "bf16x3": 6},
                        "narrow": {"tf32": 4, "bf16x3": 3}}


# ------------------------------------------------------------------------------------------------ launch arithmetic
def ring_walk(B, Hi, Wi, Ci, Co, k, mode):
    """conv_plan plus the tile walk of conv_tc_kernel: kStages of the tile shape, and for every CTA (blockIdx.x, stepping
    by the grid) each tile's split ks = tile % ksplit, decode_tile(tile / ksplit) with rot_div = max(1, grid / (nblocks *
    nphase)), the phase's k-steps it0..it1 and the (stage, phase bit) it starts at.  Returns the plan with ``stages``,
    ``starts`` (the set of start states) and ``ranges`` (the set of k-steps per tile)."""
    plan = conv_plan(B, Hi, Wi, Ci, Co, k, mode)
    bm, bn = plan["tile"]
    stages = 4 if bm * bn > 128 * 128 else 3
    nblocks, nphase, ks = Co // bn, 4 if mode == T2 else 1, plan["ksplit"]
    iters = [t * (Ci // 32) for t in ((4, 2, 2, 1) if mode == T2 else (k * k,))]
    rot_div = max(1, plan["grid"] // (nblocks * nphase))
    starts, ranges = set(), set()
    for cta in range(plan["grid"]):
        stage, ph = 0, 0
        for tile in range(cta, plan["tiles"], plan["grid"]):
            split = tile % ks
            mt, rem = divmod(tile // ks, nblocks * nphase)
            phase = 0 if nphase == 1 else (rem // nblocks + mt // rot_div) % nphase
            n = iters[phase] * (split + 1) // ks - iters[phase] * split // ks
            starts.add((stage, ph))
            ranges.add(n)
            wraps, stage = divmod(stage + n, stages)
            ph ^= wraps & 1
    return dict(plan, stages=stages, starts=starts, ranges=ranges)


def ring_label(walk):
    """What a launch reaches (see the module docstring), or None."""
    if walk["ksplit"] > 1:
        return "split-K" if len(walk["ranges"]) > 1 else None
    if not reaches(walk):
        return None
    if walk["starts"] == {(s, p) for s in range(walk["stages"]) for p in (0, 1)}:
        return "mid-ring"
    return "rounds" if {s for s, _ in walk["starts"]} == {0} else "part-ring"


def wgrad_variant(B, Hi, Wi, Ci, Co, k, mode):
    """conv_wgrad_tc.cu's host side for any variant: conv2d_wgrad_tc_supported, is_stack / is_narrow, pick_bn, the halo
    choice, wgrad_splits (one wave: base CTAs x splits <= 132) and the 32-pixel units each CTA sums."""
    Ho, Wo = out_hw(Hi, Wi, k, mode)
    Hs, Ws, Cs, Cb = (Hi, Wi, Ci, Co) if mode == T2 else (Ho, Wo, Co, Ci)
    stack = Cs == 32 and mode == S1 and k == 3
    narrow = Cs == 64 or (Cs == 32 and mode == S1 and k == 1 and Cb <= 64)
    bn = 64 if Cb % 64 == 0 else 32 if Cb % 32 == 0 else 0
    pw = min(Ws, 32)

    def pow2(v):
        return v > 0 and v & (v - 1) == 0
    supported = ((Cs % 128 == 0 or stack or narrow) and bn > 0 and pow2(Hs) and pow2(Ws) and min(Hs, Ws) >= 4
                 and (B * Hs * Ws) % 32 == 0 and (B * Hs) % (32 // pw) == 0)
    if not supported:
        return None
    units = B * Hs * Ws // 32
    base = Cb // bn if stack else (1 if narrow else Cs // 128) * (Cb // bn) * k
    splits = max(1, min(SMS // base, units))
    halo = mode == S1 and k == 3 and pw == 32
    return dict(variant="STACK" if stack else "narrow" if narrow else "wide", splits=splits,
                units_per_cta=-(-units // splits), halo=halo,
                # wgrad_tc_kernel<KW, BLOCK_N, STACK, HALO, X3, AC> without X3
                args=(k, bn, str(stack).lower(), str(halo).lower(), 2 if narrow else 4))


def launches(B, Hs, Ws, Ci, Co, k, mode):
    """The forward launch, the input-gradient launch (its adjoint) and the weight gradient of a row."""
    Hi, Wi = in_hw(Hs, Ws, mode)
    Ho, Wo = out_hw(Hi, Wi, k, mode)
    return (ring_walk(B, Hi, Wi, Ci, Co, k, mode), ring_walk(B, Ho, Wo, Co, Ci, k, ADJ[mode]),
            wgrad_variant(B, Hi, Wi, Ci, Co, k, mode))


# ------------------------------------------------------------------------------------------------ the rows
LRELU, LRELU_RT, RELU_RT = (0.2, math.sqrt(2.0), False), (0.2, math.sqrt(2.0), True), (0.0, 1.0, True)
# (step, layer, B, Hs, Ws, Ci, Co, k, mode, epilogue (slope, gain, rt in tf32) or None, (forward label, input-gradient
# label), wgrad variant, mechanism).  Hs x Ws is the SITE grid (output for S1 / S2, input for T2); channel counts are the
# model's after zero-padding to 32 (the 9-channel D input, the 6/12/24-channel condition convs, the 513-channel
# final_conv).  B is the smallest batch that reaches the forward label with a tensor-core weight gradient.
ROWS = [
    ("256", "G noise_conv.4", 4, 256, 256, 32, 128, 3, S1, None, ("mid-ring", "rounds"), "wide",
     "256x128 tiles of 9 k-steps on the 4-stage ring; wide weight gradient with Cb = 32"),
    ("256", "G noise_conv.0/.2", 2, 256, 256, 32, 32, 3, S1, RELU_RT, ("rounds", "rounds"), "STACK",
     "128x32 tiles, two CTAs per SM for rounds of 9 k-steps; fused bias + ReLU with rt; STACK weight gradient"),
    ("256", "D stem", 4, 256, 256, 32, 128, 1, S1, LRELU_RT, ("mid-ring", "part-ring"), "wide",
     "1 k-step per tile: every stage boundary is a tile boundary"),
    ("256", "D final_conv", 2, 4, 4, 544, 512, 3, S1, LRELU, ("split-K", "split-K"), "wide",
     "153 k-steps in ragged split-K ranges; the epilogue is applied in the split-K reduction"),
    ("512", "G progression.7.st_cv1", 1, 256, 256, 128, 64, 3, T2, None, ("part-ring", None), "wide",
     "T2 phases of 16/8/8/4 k-steps on the 3-stage ring, rotated from round to round: all even, so tiles start at "
     "three of the six states"),
    ("512", "G progression.7.st_cv2", 1, 512, 512, 64, 64, 3, S1, None, ("rounds", "rounds"), "narrow",
     "18 k-steps per tile; narrow weight gradient with the halo tile"),
    ("512", "G noise_conv.4", 1, 512, 512, 32, 64, 3, S1, None, ("rounds", "rounds"), "narrow",
     "9 k-steps per tile; narrow weight gradient with the halo tile and Cb = 32"),
    ("512", "D stem", 1, 512, 512, 32, 64, 1, S1, LRELU_RT, ("mid-ring", "part-ring"), "narrow",
     "1 k-step per tile on the 3-stage ring; narrow 1x1 weight gradient"),
    ("512", "D ResBlock(64->128) skip", 2, 256, 256, 64, 128, 1, S1, None, ("part-ring", "part-ring"), "wide",
     "2 k-steps per 256x128 tile: tiles start at stages 0 and 2"),
    ("1024", "G progression.8.st_cv1", 1, 512, 512, 64, 32, 3, T2, None, ("part-ring", "rounds"), "narrow",
     "T2 phases of 8/4/4/2 k-steps on the 3-stage ring for 31 rounds; narrow weight gradient with Cs = 64 (T2: the input)"),
    ("1024", "D stem", 1, 1024, 1024, 32, 32, 1, S1, LRELU_RT, ("mid-ring", "mid-ring"), "narrow",
     "1 k-step per tile; narrow weight gradient with Cs = 32"),
    ("1024", "D ResBlock(32->64).conv2", 1, 512, 512, 32, 64, 3, S2, LRELU, ("rounds", "part-ring"), "narrow",
     "stride-2 boxes at 32 channels, 9 k-steps; the input gradient is a T2 of 8/4/4/2 k-steps; narrow S2 weight gradient"),
]
ROW_IDS = [f"{r[0]}-{r[1].replace(' ', '_')}-B{r[2]}" for r in ROWS]

# (B, H, W, C, up, down, pad, gain of the model's blur kernel, mechanism): B is the smallest with which both the forward
# launch and its adjoint reach (test_layer_shapes_gpu.FIR_CASES has the C >= 128 calls)
FIR_ROWS = [
    (1, 1024, 1024, 32, 1, 1, (2, 2), 1.0, "D's blur before the 1024^2 stride-2 conv (C = 32): 1025^2 output"),
    (1, 512, 512, 64, 1, 1, (2, 2), 1.0, "D's blur before the 512^2 stride-2 conv (C = 64): 513^2 output"),
    (1, 1025, 1025, 32, 1, 1, (1, 1), 4.0, "G's blur after the 1024^2 T2 conv (C = 32)"),
    (1, 513, 513, 64, 1, 1, (1, 1), 4.0, "G's blur after the 512^2 T2 conv (C = 64)"),
    (1, 1024, 1024, 32, 1, 2, (1, 1), 1.0, "D's down2 skip at 1024^2 (C = 32); its adjoint is the up2 kernel, flip = 1"),
    (1, 512, 512, 64, 1, 2, (1, 1), 1.0, "D's down2 skip at 512^2 (C = 64); its adjoint is the up2 kernel, flip = 1"),
]
FIR_IDS = [f"{'down2' if c[5] == 2 else 'blur'}-pad{c[6][0]}-{c[1]}sq-C{c[3]}-B{c[0]}" for c in FIR_ROWS]


def row_reaches(B, Hs, Ws, Ci, Co, k, mode, label):
    fwd, _, wg = launches(B, Hs, Ws, Ci, Co, k, mode)
    return wg is not None and ring_label(fwd) == label


def fmt(w):
    return (f"{w['tile'][0]}x{w['tile'][1]}/{w['stages']} stages, {w['tiles']} tiles on {w['grid']} CTAs "
            f"({w['tiles'] / w['grid']:.2f} rounds), k-steps {sorted(w['ranges'])}"
            + (f" in {w['ksplit']} splits" if w["ksplit"] > 1 else "") + f", starts {sorted(w['starts'])}")


def test_ring_reach_cpu():
    """Each row reaches its labels with the smallest batch that does; the existing convolution rows do not reach
    mid-ring; the weight-gradient restatement agrees with test_layer_shapes_gpu.wgrad_plan on its wide rows.  Printed as a table."""
    print()
    for step, layer, B, Hs, Ws, Ci, Co, k, mode, act, (label, adj_label), variant, why in ROWS:
        fwd, adj, wg = launches(B, Hs, Ws, Ci, Co, k, mode)
        print(f"  {step}^2 {layer} ({'S1 S2 T2'.split()[mode]} {k}x{k} {Ci}->{Co}, site {Hs}x{Ws}, B={B})  -- {why}\n"
              f"      forward    {label:<9s} {fmt(fwd)}\n      input grad {str(adj_label):<9s} {fmt(adj)}\n"
              f"      wgrad {wg['variant'] if wg else None}, {wg and wg['splits']} splits x {wg and wg['units_per_cta']} units")
        assert ring_label(fwd) == label, (layer, fmt(fwd))
        assert ring_label(adj) == adj_label, (layer, fmt(adj))
        assert wg is not None and wg["variant"] == variant, (layer, wg)
        assert B == 1 or not row_reaches(B - 1, Hs, Ws, Ci, Co, k, mode, label), f"{layer}: B = {B - 1} reaches too"
    assert {r[10][0] for r in ROWS} == {"mid-ring", "part-ring", "rounds", "split-K"}
    assert {r[11] for r in ROWS} == {"wide", "STACK", "narrow"}
    assert {launches(*r[2:9])[2]["halo"] for r in ROWS if r[11] == "narrow"} == {True, False}

    print("  existing rows (test_layer_shapes_gpu.CONV_CASES, test_conv_tc_large_gpu.CASES): forward / input gradient")
    existing = [(B, Hs, Ws, Ci, Co, 3, mode) for B, Hs, Ws, Ci, Co, mode, *_ in LS.CONV_CASES] + list(LARGE_CASES)
    for B, Hs, Ws, Ci, Co, k, mode in existing:
        walks = launches(B, Hs, Ws, Ci, Co, k, mode)[:2]
        print(f"    {'S1 S2 T2'.split()[mode]} {Ci}->{Co} site {Hs}x{Ws} B={B}: "
              + " / ".join(f"{ring_label(w)}: {fmt(w)}" for w in walks))
        assert all(ring_label(w) != "mid-ring" for w in walks), (B, Hs, Ws, Ci, Co, k, mode)
    for B, Hs, Ws, Ci, Co, mode, *_ in LS.CONV_CASES:     # the wide variant, as test_layer_shapes_gpu restates it
        Hi, Wi = in_hw(Hs, Ws, mode)
        wg = wgrad_variant(B, Hi, Wi, Ci, Co, 3, mode)
        assert wg["variant"] == "wide" and wgrad_plan(B, Hi, Wi, Ci, Co, 3, mode) == \
            {key: wg[key] for key in ("splits", "units_per_cta")}

    for B, H, W, C, up, down, pad, _, why in FIR_ROWS:
        plans = fir_launches(B, H, W, C, up, down, pad)
        print("  fir " + ", ".join(f"{p['kernel']} {p['tiles']} tiles on {p['grid']} CTAs ({p['tiles'] / p['grid']:.2f} rounds)"
                                   for p in plans) + f"  -- {why}")
        assert all(p is not None and reaches(p) for p in plans), (why, plans)
        assert B == 1 or not all(reaches(p) for p in fir_launches(B - 1, H, W, C, up, down, pad)), why
    assert fir_plan(1, 1024, 1024, 32, 512, 512, 1, 2, 1)["kernel"] == "upfirdn2d_fir4_pipe_kernel<2>"
    assert {fir_launches(*c[:7])[1]["kernel"] for c in FIR_ROWS if c[5] == 2} == {"upfirdn2d_up2_pipe_kernel"}


# ------------------------------------------------------------------------------------------------ convolutions
@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=ROW_IDS)
def test_conv_ring_at_layer_shape(cuda, tc_precision, row):
    """Forward with the model's epilogue, input gradient and weight gradient against float64; the launch plan through
    the library."""
    from gif_b200 import ops
    from gif_b200._lib import lib
    step, layer, B, Hs, Ws, Ci, Co, k, mode, act, _, variant, why = row
    precision = tc_precision
    impl = 3 if precision == "bf16x3" else 2
    Hi, Wi = in_hw(Hs, Ws, mode)
    Ho, Wo = out_hw(Hi, Wi, k, mode)
    fwd, adj, wg = launches(B, Hs, Ws, Ci, Co, k, mode)
    for plan, args in ((fwd, (B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, 0)), (adj, (B, Ho, Wo, Co, Hi, Wi, Ci, k, ADJ[mode], 1))):
        part = plan["ksplit"] * B * args[4] * args[5] * args[6] * 4 + 256 if plan["ksplit"] > 1 else 0
        assert lib.gifb200_conv2d_workspace_bytes(*args, impl) == staged_weight_bytes(Ci, Co, k) + part, (layer, plan)
    assert lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl) == impl
    assert lib.gifb200_conv2d_wgrad_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl) == \
        wg["splits"] * k * k * Co * Ci * 4 + 256

    g = torch.Generator(device="cuda").manual_seed(int(step) + B * 1000 + Hs + Ci * 7 + Co * 3 + k + mode)
    x = torch.randn(B, Hi, Wi, Ci, device=cuda, generator=g)
    w = torch.randn(k * k, Co, Ci, device=cuda, generator=g) / math.sqrt(k * k * Ci)
    gy = torch.randn(B, Ho, Wo, Co, device=cuda, generator=g)
    bias = None if act is None else 0.1 * torch.randn(Co, device=cuda, generator=g)
    if precision == "tf32":
        x, w, gy = (ops._round_tf32_raw(t) for t in (x, w, gy))
    rt = act is not None and act[2] and precision == "tf32"     # the model rounds these outputs in tf32 mode only

    x3 = "true" if precision == "bf16x3" else "false"
    want = {f"{p['tile'][0]},{p['tile'][1]},{x3}" for p in (fwd, adj)}
    want_wg = {",".join(str(a) for a in wg["args"][:4] + (x3, wg["args"][4]))}
    out = {}

    def run():
        with tensor_cores_only(precision):
            leaves = [x.clone().requires_grad_(True), w.clone().requires_grad_(True)]
            if act is None:
                out["y"] = ops.conv2d(leaves[0], leaves[1], k, mode)
            else:
                leaves.append(bias.clone().requires_grad_(True))
                out["y"] = ops.conv2d_bias_act(leaves[0], leaves[1], leaves[2], k, mode, act[0], act[1], rt=rt)
            out["g"] = torch.autograd.grad(out["y"], leaves, gy)

    names = kernel_names(run, lambda ns: want <= template_args(ns, "conv_tc_kernel")
                         and template_args(ns, "wgrad_tc_kernel") == want_wg)
    tiles = template_args(names, "conv_tc_kernel")
    assert want <= tiles, (why, want, tiles)
    assert template_args(names, "wgrad_tc_kernel") == want_wg, (variant, want_wg, template_args(names, "wgrad_tc_kernel"))

    y = out["y"]
    x64, w64, gy64 = x.double(), w.double(), gy.double()
    if act is None:
        yr, gpre, gpre64 = ref_conv(x64, w64, k, mode), gy, gy64
    else:
        slope, gain, _ = act
        if rt:
            with torch.no_grad():
                y_plain = ops.conv2d_bias_act(x, w, bias, k, mode, slope, gain)
            assert torch.equal(y, ops._round_tf32_raw(y_plain)), "rt: not the rounding of the unrounded output"
            y = y_plain
        m = lrelu_mask(y, slope, gain)
        yr = m * (ref_conv(x64, w64, k, mode) + bias.double())
        # the pre-activation gradient as the fused activation backward forms it: gy * gain * (y > 0 ? 1 : slope) in fp32;
        # rounded to tf32 in tf32 mode, where both backward convolutions read the rounded values
        gpre = gy * gain * torch.full_like(y, slope).masked_fill_(y > 0, 1.0)
        if precision == "tf32":
            gpre = ops._round_tf32_raw(gpre)
        gpre64 = gpre.double() if precision == "tf32" else m * gy64
    xr, wr = x64.requires_grad_(True), w64.requires_grad_(True)
    gxr, gwr = torch.autograd.grad(ref_conv(xr, wr, k, mode), (xr, wr), gpre64)
    old = ops.CONV_IMPL
    ops.CONV_IMPL = 1
    try:
        gw_simt = ops._wgrad_raw(x, gpre, k, mode, False, False)
    finally:
        ops.CONV_IMPL = old

    print(f"\n  {step}^2 {layer}: {why}")
    assert_close("y", y, yr, precision, bar=BAR[precision])
    assert_close("gx", out["g"][0], gxr, precision, bar=BAR[precision])
    if act is not None:
        # the bias gradient sums the unrounded pre-activation gradient
        assert_close("gb", out["g"][2], (m * gy64).sum((0, 1, 2)), precision, lower=False, bar=BAR[precision])
    assert_close("gw simt fp32", gw_simt, gwr, "fp32", lower=False, bar=BAR[precision])
    steps = wg["units_per_cta"] * WGRAD_STEPS_PER_UNIT[variant][precision]
    print(f"  gw ({variant}): {wg['units_per_cta']} units = {steps} accumulate steps per register: bar "
          f"{BAR[precision]:.0e} + {steps} x 2^-24")
    assert_close("gw", out["g"][1], gwr, precision, bar=BAR[precision] + steps * 2.0 ** -24)


# ------------------------------------------------------------------------------------------------ FIR
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["blur", "random"])
@pytest.mark.parametrize("B,H,W,C,up,down,pad,gain,why", FIR_ROWS, ids=FIR_IDS)
def test_fir_at_narrow_layer_shape(cuda, fp32_mode, B, H, W, C, up, down, pad, gain, why, kind):
    """test_layer_shapes_gpu's FIR check (forward and autograd adjoint in fp32 against float64 at FIR_BAR, the pipe
    kernel of both calls from the profile) at the 32- and 64-channel calls."""
    assert FIR_BAR == 1e-5
    LS.test_fir_at_layer_shape(cuda, fp32_mode, B, H, W, C, up, down, pad, gain, why, kind)
