"""GPU: generator and discriminator at 512^2 and 1024^2 -- G forward and first derivatives (with a full-size condition and
with a 256^2 condition that the pyramid upsamples), D scores, R1 penalty and gradients -- in fp32, tf32 and bf16x3.  At
512^2 the reference is tests/golden/highres.npz (the unmodified reference modules in float64, tools/make_highres_golden.py);
at 1024^2 it is the in-repo oracle evaluated live in float64 on the device, with F.interpolate as its pyramid (what the
reference does; pinned against the reference at 512^2 in tests/golden/HIGHRES_ORACLE_VS_REFERENCE.txt).  The sampled
weights include the narrow (32- / 64-channel) layers whose weight gradients run on the narrow tensor-core variant."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu
from oracle import stylegan2_oracle as O

pytestmark = pytest.mark.gpu

MODES = {  # forward, gradient (l2) and R1 bars; bf16x3 carries the 256^2 model tests' bars
    "fp32": dict(fwd=1e-4, grad=5e-3, r1=5e-4),
    "tf32": dict(fwd=3e-3, grad=5e-2, r1=3e-2),
    "bf16x3": dict(fwd=2e-4, grad=8e-3, r1=1e-3),
}


def l2rel(a, b):
    a = np.asarray(a, np.float64).ravel()
    b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def f64(sd, dev):
    return {k: v.to(dev, torch.float64) for k, v in sd.items()}


def bilinear(c, size):
    return F.interpolate(c, size=(size, size), mode="bilinear", align_corners=False)


@pytest.fixture()
def precision():
    from gif_b200 import ops
    old = ops.get_precision()
    yield ops.set_precision
    ops.set_precision(old)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("res,cond_res", [(512, 512), (512, 256), (1024, 1024), (1024, 256)])
def test_generator_highres_vs_oracle(cuda, precision, monkeypatch, mode, res, cond_res):
    from gif_b200.model.stg2_generator import StyledGenerator
    precision(mode)
    step = int(np.log2(res)) - 2
    monkeypatch.setattr(O, "cond_pyramid_level", bilinear)      # the oracle's pyramid, extended to upsampling levels
    vocab = 16
    sd = gu.seeded_state_dict(gu.g_shapes(vocab), 11)
    G = StyledGenerator(embedding_vocab_size=vocab, rendered_flame_ascondition=True, normal_maps_as_cond=True)
    G.load_state_dict(sd)
    G = G.to(cuda)
    cond = gu.rand_uniform((2, 6, cond_res, cond_res), 12).to(cuda)
    idx = gu.randint(vocab, (2,), 13).to(cuda)
    gy = gu.randn((2, 3, res, res), 14).to(cuda)
    names = [f"generator.progression.{step}.st_cv1.conv.weight", f"generator.progression.{step}.st_cv2.conv.weight",
             f"generator.progression.{step}.st_cv2.noise.noise_conv.4.weight", "generator.progression.5.st_cv2.conv.weight"]
    cond_g = cond.clone().requires_grad_(True)
    img = G(cond_g, step=step, input_indices=idx)[0]
    assert tuple(img.shape) == (2, 3, res, res)
    named = dict(G.named_parameters())
    grads = torch.autograd.grad((img * gy).sum(), [cond_g] + [named[n] for n in names])
    bar = MODES[mode]
    if res == 512:
        g = gu.load_golden("highres.npz")
        tag = f"g512_c{cond_res}"
        s, _ = gu.sample(img, 8192, 5)
        assert np.abs(s - g[tag + "_img"]).max() / float(g[tag + "_img_absmax"]) < bar["fwd"]
        for n, gr in zip(["cond"] + names, grads):
            assert l2rel(gu.sample(gr, 4096, 6)[0], g[f"{tag}_g_{n}"]) < bar["grad"], n
        return

    sd64 = {k: v.requires_grad_(k in names) for k, v in f64(sd, cuda).items()}
    cond64 = cond.double().requires_grad_(True)
    ref = O.generator_forward(cond64, idx, sd64, step)
    ref_grads = torch.autograd.grad((ref * gy.double()).sum(), [cond64] + [sd64[n] for n in names])
    assert gu.rel_err(img.detach().cpu().numpy(), ref.detach().cpu().numpy()) < bar["fwd"]
    for n, a, b in zip(["cond"] + names, grads, ref_grads):
        assert l2rel(a.cpu().numpy(), b.cpu().numpy()) < bar["grad"], n


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("size", [512, 1024])
def test_discriminator_highres_r1_vs_oracle(cuda, precision, mode, size):
    from gif_b200 import losses
    from gif_b200.model.stg2_discriminator import Discriminator
    precision(mode)
    sd = gu.seeded_state_dict(gu.d_shapes(size), 21)
    D = Discriminator(size, num_color_chnls=9)
    D.load_state_dict(sd)
    D = D.to(cuda)
    names = ["convs.0.0.weight", "convs.1.conv1.0.weight", "convs.1.conv2.1.weight", "convs.1.skip.1.weight",
             "final_conv.0.weight"]
    img = gu.rand_uniform((4, 3, size, size), 22).to(cuda)
    cond = gu.rand_uniform((4, 6, size, size), 23).to(cuda)
    x = img.clone().requires_grad_(True)
    scores, _ = D([x], condition=cond)
    pen = losses.grad_penalty_loss([x], scores, step=None)
    named = dict(D.named_parameters())
    grads = torch.autograd.grad(F.softplus(-scores).mean() + pen.mean(), [named[n] for n in names])

    if size == 512:
        # With these seeded weights the 512^2 scores are sums that cancel to ~1e-3, so their relative error measures the
        # cancellation as much as the kernels.  Measured on an H100 against this golden: torch's own float32 convolutions
        # of the oracle are 3.6e-4 off (the reference's float32 on the CPU, recorded in the golden, 6.5e-5), this
        # project's exact-fp32 kernels 2.6e-4, and torch's tf32 convolutions 6.7e-2.  The score bar is the fixed one, but
        # not below 3x torch's float32 error (1.1e-3); tf32 gets 0.1.  The R1 bars are the fixed ones.
        g = gu.load_golden("highres.npz")
        ref_s, ref_p = g["d512_scores"], g["d512_r1"]
        ref_grads = [g["d512_g_" + n] for n in names]
        fwd_bar = 0.1 if mode == "tf32" else max(MODES[mode]["fwd"], 3 * 3.6e-4)
        r1_bar = MODES[mode]["r1"]
        grads = [gu.sample(gr, 4096, 7)[0] for gr in grads]
    else:
        sd64 = {k: v.requires_grad_(k in names) for k, v in f64(sd, cuda).items()}
        x64 = img.double().requires_grad_(True)
        s64 = O.discriminator_forward(x64, cond.double(), sd64, size)
        p64 = O.r1_penalty(s64, x64)
        ref_grads = torch.autograd.grad(F.softplus(-s64).mean() + p64.mean(), [sd64[n] for n in names])
        ref_s, ref_p = s64.detach().cpu().numpy(), p64.detach().cpu().numpy()
        ref_grads = [r.cpu().numpy() for r in ref_grads]
        grads = [gr.cpu().numpy() for gr in grads]
        fwd_bar, r1_bar = MODES[mode]["fwd"], MODES[mode]["r1"]
    e_s = gu.rel_err(scores.detach().cpu().numpy(), ref_s)
    e_p = gu.rel_err(pen.detach().cpu().numpy(), ref_p)
    print(f"D{size} {mode}: scores {e_s:.2e} (bar {fwd_bar:.1e}), R1 {e_p:.2e} (bar {r1_bar:.1e})")
    assert e_s < fwd_bar
    assert e_p < r1_bar
    for n, a, b in zip(names, grads, ref_grads):
        assert l2rel(a, b) < MODES[mode]["grad"], n
