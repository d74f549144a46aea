"""GPU parity tests of the generator / discriminator / R1 / PPL against the reference goldens and the oracle, in the
three precision modes of gif_b200.ops (tools/precision_report.py measures the table):

    quantity (vs reference golden)        fp32 SIMT    tf32 wgmma      bf16x3 wgmma        bar of BASELINE.json
    G 32^2 / 256^2 forward (max-rel)      3.5e-6       0.9-1.2e-3      4.7e-5 / 8.8e-5     1e-3
    D 64^2 / 256^2 scores                 1.4e-6       6.1e-4          3.9e-5 / 6.1e-5     1e-3
    R1 penalty (double backward)          3.1e-5       1.3e-2          3.3e-4              1e-3
    network gradients, L2 vs fp64         1.0-2.1e-3   2.0-3.2e-2      3.4-4.7e-3          (reference's own fp32: 0.95e-3)

bf16x3 (the error-compensated contraction) is the mode that holds the 1e-3 bar end to end -- forward, scores and the R1
penalty -- and it is the mode bench.py headlines; plain tf32 meets it per operator (tests/test_ops_tc_golden_gpu.py) but
not through 7-14 chained layers, and is reported as the faster, lower-precision option.

Network-level GRADIENTS are compared with the reference evaluated in float64 (``*_f64`` goldens).  Through ~14 leaky
ReLUs the gradient is only piecewise continuous: a pre-activation within the forward error eps of zero flips its mask, so
a forward error eps turns into an L2 gradient error ~sqrt(eps) whatever the arithmetic.  The reference's OWN fp32 gradient
differs from its fp64 value by 0.95e-3 (L2, tests/golden/ORACLE_VS_REFERENCE.txt: eps ~1e-6); this repo's exact-fp32 path
sits at 1.0-2.1e-3, bf16x3 (eps ~4e-5) at 3.4-4.7e-3, tf32 (eps ~1e-3) at 2-3e-2 -- the sqrt law, not an arithmetic
defect (every operator's own backward is inside its forward bar on identical inputs, test_ops_tc_golden_gpu.py).  Bars:
fp32 max(1e-3, 3x the reference's floor) resp. 5e-3 for G, bf16x3 8e-3, tf32 5e-2.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu
from oracle import stylegan2_oracle as O

pytestmark = pytest.mark.gpu


def l2rel(a, b):
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def make_g(cuda, seed=1, vocab=100):
    from gif_b200.model.stg2_generator import StyledGenerator
    G = StyledGenerator(embedding_vocab_size=vocab, rendered_flame_ascondition=True, normal_maps_as_cond=True,
                        core_tensor_res=4, n_mlp=8)
    sd = gu.seeded_state_dict(gu.g_shapes(vocab), seed)
    G.load_state_dict(sd)
    return G.to(cuda), sd


def make_d(cuda, size, seed):
    from gif_b200.model.stg2_discriminator import Discriminator
    D = Discriminator(size, num_color_chnls=9)
    sd = gu.seeded_state_dict(gu.d_shapes(size), seed)
    D.load_state_dict(sd)
    return D.to(cuda), sd


G_PNAMES = ["generator.progression.2.st_cv1.conv.weight", "generator.progression.3.st_cv2.conv.modulation.weight",
            "generator.progression.1.st_cv2.noise.noise_conv.4.weight", "generator.to_rgb.2.conv.weight",
            "generator.to_rgb.3.bias", "z_to_w.3.weight", "generator.const_input.input",
            "generator.progression.3.st_cv1.activate.bias"]
D_PNAMES = ["convs.0.0.weight", "convs.1.conv1.0.weight", "convs.2.conv2.1.weight", "convs.3.skip.1.weight",
            "convs.2.conv2.2.bias", "final_conv.0.weight", "final_linear.0.weight", "final_linear.1.bias"]


@pytest.mark.parametrize("mode,tol_fwd,tol_grad", [("fp32", 5e-5, 5e-3), ("tf32", 3e-3, 5e-2), ("bf16x3", 2e-4, 8e-3)])
def test_generator_step3_golden(cuda, mode, tol_fwd, tol_grad):
    from gif_b200 import ops
    ops.set_precision(mode)
    try:
        g = gu.load_golden("generator.npz")
        G, _ = make_g(cuda)
        cond = gu.rand_uniform((2, 6, 32, 32), 40).to(cuda).requires_grad_(True)
        idx = gu.randint(100, (2,), 41).to(cuda)
        img = G(cond, step=3, input_indices=idx)[0]
        assert tuple(img.shape) == (2, 3, 32, 32)
        assert gu.rel_err(img.detach().cpu().numpy(), g["s3_img"]) < tol_fwd
        gy = gu.randn(tuple(img.shape), 42).to(cuda)
        named = dict(G.named_parameters())
        grads = torch.autograd.grad((img * gy).sum(), [cond] + [named[n] for n in G_PNAMES])
        assert l2rel(grads[0].cpu().numpy(), g["s3_gcond_f64"]) < tol_grad, "grad cond"
        for n, gr in zip(G_PNAMES, grads[1:]):
            s, tot = gu.sample(gr, 2048, 2)
            assert l2rel(s, g["s3_g64_" + n]) < tol_grad, n
        # float-z path (gen.py:272-273)
        with torch.no_grad():
            img_z = G(cond.detach(), step=3, input_indices=gu.randn((2, 512), 43).to(cuda))[0]
        assert gu.rel_err(img_z.cpu().numpy(), g["s3_img_z"]) < tol_fwd
    finally:
        ops.set_precision("tf32")


@pytest.mark.parametrize("mode,tol", [("fp32", 1e-4), ("tf32", 3e-3), ("bf16x3", 5e-4)])
def test_generator_256_golden(cuda, mode, tol):
    """BASELINE configs[1] shape (256^2, step 6), B=2: sampled reference output."""
    from gif_b200 import ops
    ops.set_precision(mode)
    try:
        g = gu.load_golden("generator.npz")
        G, _ = make_g(cuda)
        with torch.no_grad():
            img = G(gu.rand_uniform((2, 6, 256, 256), 44).to(cuda), step=6, input_indices=gu.randint(100, (2,), 45).to(cuda))[0]
        assert tuple(img.shape) == (2, 3, 256, 256)
        s, tot = gu.sample(img, 8192, 3)
        assert np.abs(s - g["s6_sample"]).max() / float(g["s6_absmax"]) < tol
        assert abs(tot - float(g["s6_sum"])) / (float(g["s6_absmax"]) * math.sqrt(img.numel())) < 10 * tol
    finally:
        ops.set_precision("tf32")


@pytest.mark.parametrize("mode,tol_fwd", [("fp32", 5e-5), ("tf32", 3e-3), ("bf16x3", 2e-4)])
def test_discriminator_64_r1_golden(cuda, mode, tol_fwd):
    """Discriminator(64, 9ch) B=8: scores, R1 penalty (double backward), all gradients of softplus + R1."""
    from gif_b200 import losses, ops
    ops.set_precision(mode)
    try:
        g = gu.load_golden("discriminator.npz")
        D, _ = make_d(cuda, 64, 2)
        img = gu.rand_uniform((8, 3, 64, 64), 50).to(cuda).requires_grad_(True)
        cond = gu.rand_uniform((8, 6, 64, 64), 51).to(cuda).requires_grad_(True)
        scores, _ = D([img], condition=cond)
        assert tuple(scores.shape) == (8, 1)
        pen = losses.grad_penalty_loss([img], scores, step=None)
        assert gu.rel_err(scores.detach().cpu().numpy(), g["d64_scores"]) < tol_fwd
        # R1 penalty: 1e-3 (BASELINE.json's bar) in the exact and the compensated mode; plain tf32 cannot hold it (1.3e-2)
        assert gu.rel_err(pen.detach().cpu().numpy(), g["d64_r1"]) < {"fp32": 5e-4, "bf16x3": 1e-3, "tf32": 3e-2}[mode]
        loss = F.softplus(-scores).mean() + pen.mean()
        named = dict(D.named_parameters())
        grads = torch.autograd.grad(loss, [img, cond] + [named[n] for n in D_PNAMES])
        floor = float(g["d64_gimg_ref32_l2err"])          # the reference's own fp32-vs-fp64 error
        tol = {"fp32": max(1e-3, 3 * floor), "bf16x3": 8e-3, "tf32": 5e-2}[mode]
        assert l2rel(grads[0].cpu().numpy(), g["d64_gimg_f64"]) < tol, "grad img"
        assert l2rel(grads[1].cpu().numpy(), g["d64_gcond_f64"]) < tol, "grad cond"
        for n, gr in zip(D_PNAMES, grads[2:]):
            s, _ = gu.sample(gr, 2048, 4)
            assert l2rel(s, g["d64_g64_" + n]) < tol, n
    finally:
        ops.set_precision("tf32")


@pytest.mark.parametrize("mode,tol", [("fp32", 1e-4), ("tf32", 3e-3), ("bf16x3", 3e-4)])
def test_discriminator_256_golden(cuda, mode, tol):
    from gif_b200 import ops
    ops.set_precision(mode)
    try:
        g = gu.load_golden("discriminator.npz")
        D, _ = make_d(cuda, 256, 3)
        with torch.no_grad():
            scores, none = D([gu.rand_uniform((4, 3, 256, 256), 52).to(cuda)],
                             condition=gu.rand_uniform((4, 6, 256, 256), 53).to(cuda))
        assert none is None
        assert gu.rel_err(scores.cpu().numpy(), g["d256_scores"]) < tol
    finally:
        ops.set_precision("tf32")


@pytest.mark.parametrize("mode,tol_val,tol_grad", [("fp32", 1e-3, 1e-2), ("bf16x3", 2e-3, 3e-2), ("tf32", 3e-2, 3e-1)])
def test_path_length_regulariser_vs_oracle(cuda, mode, tol_val, tol_grad):
    """PPL (parity UNPINNED in the reference, SURVEY 8 L2): the adopted rule, CUDA path vs oracle autograd, incl. the
    gradient of the penalty w.r.t. a generator weight (needs the double backward of every G op) -- in all three precision
    modes (the penalty is a second-order quantity: ||d img / d w|| through 5 modulated convolutions and their activations)."""
    from gif_b200 import losses, ops
    ops.set_precision(mode)
    try:
        _ppl_case(cuda, mode, tol_val, tol_grad)
    finally:
        ops.set_precision("tf32")


def _ppl_case(cuda, mode, tol_val, tol_grad):
    from gif_b200 import losses
    G, sd = make_g(cuda)
    cond = gu.rand_uniform((2, 6, 16, 16), 60)
    idx = gu.randint(100, (2,), 61)
    noise = gu.randn((2, 3, 16, 16), 62)
    pname = "generator.progression.1.st_cv2.conv.weight"
    # oracle
    sd_o = {k: v.clone().requires_grad_(k == pname) for k, v in sd.items()}
    pen_o, ema_o, len_o = O.path_length_penalty(cond, idx, sd_o, noise, pl_mean=0.0, step=2)
    (g_o,) = torch.autograd.grad(pen_o, sd_o[pname])
    # CUDA path
    reg = losses.PathLengthRegularizor()
    pen = reg.path_length_reg(G, step=2, alpha=1, input_indices=idx.to(cuda), cond=cond.to(cuda), pl_noise=noise.to(cuda))
    (g_c,) = torch.autograd.grad(pen, dict(G.named_parameters())[pname])
    e_pen = abs(float(pen.detach()) - float(pen_o.detach())) / abs(float(pen_o.detach()))
    e_ema = abs(float(reg.pl_moving_mean) - float(ema_o)) / abs(float(ema_o))
    e_g = l2rel(g_c.cpu().numpy(), g_o.numpy())
    print(f"PPL [{mode}]: penalty {e_pen:.2e}  ema {e_ema:.2e}  grad L2 {e_g:.2e}")
    assert e_pen < tol_val and e_ema < tol_val
    assert e_g < tol_grad      # mask-flip noise floor of a double backward, see module docstring


def test_drop_in_module_names():
    import gif_b200
    gif_b200.install_as_reference_modules(data_parallel=False)
    from model.stg2_generator import StyledGenerator  # noqa: F401
    from model.stg2_discriminator import Discriminator  # noqa: F401
    from model.stylegan2_common_layers import (Blur, ConvLayer, EqualConv2d, EqualLinear, FusedLeakyReLU,  # noqa: F401
                                               ModulatedConv2d, NoiseInjection, ResBlock, StyledConv, ToRGB,
                                               Upsample, upfirdn2d, make_kernel)
