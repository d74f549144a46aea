#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY (build container) -- goldens for the TENSOR-CORE shapes of the contraction operators.

``tests/golden/modconv.npz`` / ``ops.npz`` hold small shapes (Co = 16, Ci = 16 ...) that the tensor-core kernels do not take, so
they pin the exact-fp32 SIMT path only.  This script evaluates the UNMODIFIED reference modules (oracle/ref_import.py) on
shapes the tensor-core path DOES take -- channels multiples of 32, power-of-two site grids, incl. the north-star layer
ModulatedConv2d(128,128,3) at 256^2 and BASELINE.json configs[0] -- in float64 (the truth the 1e-3 bar is read against)
and in float32 (the reference's own rounding floor, stored as ``*_floor``) -> tests/golden/ops_tc.npz.
Consumed by tests/test_ops_tc_golden_gpu.py, which runs every case in tf32, bf16x3 and fp32 mode."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import golden_util as gu  # noqa: E402
from oracle import ref_import  # noqa: E402

R = ref_import.load()
OUT = {}


def l2rel(a, b):
    a, b = a.detach().double().reshape(-1), b.detach().double().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def record(tag, names, tensors64, tensors32, sample=None):
    sample = sample or 16384
    """Stores float64 results (full, or a fixed sample + norm for big ones) and the fp32-vs-fp64 L2 floor."""
    for n, t64, t32 in zip(names, tensors64, tensors32):
        if sample and t64.numel() > sample:
            OUT[f"{tag}_{n}"] = gu.sample(t64, sample, 9)[0]
            OUT[f"{tag}_{n}_absmax"] = np.array(float(t64.detach().abs().max()))
        else:
            OUT[f"{tag}_{n}"] = t64.detach().numpy()
        OUT[f"{tag}_{n}_floor"] = np.array(l2rel(t32, t64))


def modconv(tag, ci, co, k, demod, up, b, hw, sample=None):
    res = []
    for dt in (torch.float64, torch.float32):
        m = R.cl.ModulatedConv2d(ci, co, k, 512, demodulate=demod, upsample=up)
        m.weight.data = gu.randn((1, co, ci, k, k), 120)
        m.modulation.weight.data = gu.randn((ci, 512), 121)
        m.modulation.bias.data = 1.0 + 0.1 * gu.randn((ci,), 122)
        m = m.to(dt)
        x = gu.randn((b, ci, hw, hw), 123).to(dt).requires_grad_(True)
        st = gu.randn((b, 512), 124).to(dt).requires_grad_(True)
        y = m(x, st)
        gy = gu.randn(tuple(y.shape), 125).to(dt)
        grads = torch.autograd.grad((y * gy).sum(), [x, st, m.weight, m.modulation.weight, m.modulation.bias])
        res.append([y] + list(grads))
    record(tag, "y gx gstyle gw gmodw gmodb".split(), res[0], res[1], sample)
    print(tag, "fp32 floors:", [f"{OUT[f'{tag}_{n}_floor']:.1e}" for n in "y gx gstyle gw gmodw gmodb".split()])


def equal_conv(tag, ci, co, k, stride, pad, b, hw):
    res = []
    for dt in (torch.float64, torch.float32):
        m = R.cl.EqualConv2d(ci, co, k, stride=stride, padding=pad, bias=True)
        m.weight.data = gu.randn((co, ci, k, k), 130)
        m.bias.data = 0.1 * gu.randn((co,), 131)
        m = m.to(dt)
        x = gu.randn((b, ci, hw, hw), 132).to(dt).requires_grad_(True)
        y = m(x)
        gy = gu.randn(tuple(y.shape), 133).to(dt)
        grads = torch.autograd.grad((y * gy).sum(), [x, m.weight, m.bias])
        res.append([y] + list(grads))
    record(tag, "y gx gw gb".split(), res[0], res[1])
    print(tag, "fp32 floors:", [f"{OUT[f'{tag}_{n}_floor']:.1e}" for n in "y gx gw gb".split()])


def res_block(tag, ci, co, b, hw):
    """ResBlock = ConvLayer(3x3) -> ConvLayer(blur, 3x3 stride 2) + skip ConvLayer(blur, 1x1 stride 2)  (cl.py:802-820)."""
    res = []
    shapes = None
    for dt in (torch.float64, torch.float32):
        m = R.cl.ResBlock(ci, co)
        sd = m.state_dict()
        g = torch.Generator().manual_seed(140)
        for kk in sd:
            if kk.endswith("kernel"):
                continue
            sd[kk] = torch.randn(sd[kk].shape, generator=g) * (0.1 if "bias" in kk else 1.0)
        m.load_state_dict(sd)
        shapes = {kk: tuple(v.shape) for kk, v in sd.items()}
        m = m.to(dt)
        x = gu.randn((b, ci, hw, hw), 141).to(dt).requires_grad_(True)
        y = m(x)
        gy = gu.randn(tuple(y.shape), 142).to(dt)
        named = dict(m.named_parameters())
        pn = ["conv1.0.weight", "conv1.1.bias", "conv2.1.weight", "conv2.2.bias", "skip.1.weight"]
        grads = torch.autograd.grad((y * gy).sum(), [x] + [named[n] for n in pn])
        res.append([y] + list(grads))
    record(tag, ["y", "gx"] + ["g_" + n for n in pn], res[0], res[1])
    print(tag, "fp32 floors:", [f"{OUT[k]:.1e}" for k in OUT if k.startswith(tag) and k.endswith("_floor")])


def noise_injection(tag, cin, cout, b, hw):
    """NoiseInjection (cl.py:388-431): image + Conv3x3(ReLU(Conv3x3(ReLU(Conv3x3(cond))))) -- where the FLAME condition
    enters the generator; small-K convolutions (6 -> 12 -> 24 -> Co) that the tensor-core modes run zero-padded to 32."""
    res = []
    pn = ["noise_conv.0.weight", "noise_conv.0.bias", "noise_conv.2.weight", "noise_conv.4.weight", "noise_conv.4.bias"]
    for dt in (torch.float64, torch.float32):
        m = R.cl.NoiseInjection(cin, cout)
        sd = m.state_dict()
        g = torch.Generator().manual_seed(150)
        for kk in sd:
            sd[kk] = torch.randn(sd[kk].shape, generator=g) * (0.05 if "bias" in kk else 0.3)
        m.load_state_dict(sd)
        m = m.to(dt)
        img = gu.randn((b, cout, hw, hw), 151).to(dt).requires_grad_(True)
        cond = gu.rand_uniform((b, cin, hw, hw), 152).to(dt).requires_grad_(True)
        y = m(img, cond)
        gy = gu.randn(tuple(y.shape), 153).to(dt)
        named = dict(m.named_parameters())
        grads = torch.autograd.grad((y * gy).sum(), [img, cond] + [named[n] for n in pn])
        res.append([y] + list(grads))
    record(tag, ["y", "gimg", "gcond"] + ["g_" + n for n in pn], res[0], res[1])
    print(tag, "fp32 floors:", [f"{OUT[k]:.1e}" for k in OUT if k.startswith(tag) and k.endswith("_floor")])


def main():
    torch.manual_seed(0)
    modconv("mc_plain", 64, 64, 3, True, False, 3, 16)
    modconv("mc_up", 64, 32, 3, True, True, 3, 8)
    modconv("mc_rgb", 64, 3, 1, False, False, 3, 16)
    modconv("mc_northstar", 128, 128, 3, True, False, 2, 256, sample=8192)      # SURVEY 8d config 3b (B = 2)
    modconv("mc_config1", 512, 512, 3, True, False, 4, 64, sample=8192)         # BASELINE.json configs[0], with gradients
    equal_conv("ec_s1", 64, 128, 3, 1, 1, 2, 32)
    equal_conv("ec_s2", 64, 64, 3, 2, 0, 2, 33)
    equal_conv("ec_1x1", 64, 32, 1, 1, 0, 2, 32)
    res_block("rb", 64, 128, 2, 32)
    noise_injection("ni", 6, 64, 2, 32)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ops_tc.npz"), **OUT)
    print("wrote tests/golden/ops_tc.npz:", len(OUT), "arrays,",
          os.path.getsize(os.path.join(ROOT, "tests", "golden", "ops_tc.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
