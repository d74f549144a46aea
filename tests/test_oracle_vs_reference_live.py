"""CPU: the oracle restatement against the unmodified reference modules over randomised configurations (the other goldens
pin fixed cases; this sweeps shapes, pads, flags).  The reference's outputs for these seeded inputs are stored in
tests/golden/reference_live.npz (oracle/make_live_golden.py; inputs: tests/live_cases.py).  fp64 where the reference allows
it (its make_kernel is fp32-only: cl.py:83-91), bar 1e-11."""
import pytest
import torch

import golden_util as gu
import live_cases as LC
from oracle import stylegan2_oracle as O

DT = torch.float64


def _g(key):
    return torch.from_numpy(gu.load_golden("reference_live.npz")[key])


def _close(a, b, tol=1e-11):
    a, b = a.detach(), b.detach()
    err = float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)
    assert err < tol, err


@pytest.mark.parametrize("seed", range(6))
def test_upfirdn2d_random_configs(seed):
    cases = LC.upfirdn_cases(seed)
    assert cases
    for j, (x, k, up, down, pad) in enumerate(cases):
        _close(O.upfirdn2d(x, k, up, down, pad), _g(f"upfirdn_{seed}_{j}"))


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("upsample", [False, True])
@pytest.mark.parametrize("demod", [True, False])
def test_modulated_conv2d_random_configs(seed, upsample, demod):
    c = LC.modconv_case(seed, upsample, demod)
    key = f"modconv_{seed}_{int(upsample)}_{int(demod)}"
    y_o = O.modulated_conv2d(c["x"], c["s"], c["weight"], c["mod_weight"], c["mod_bias"], demodulate=demod,
                             upsample=upsample, blur_kernel=_g(key + "_blur") if upsample else None)
    _close(y_o, _g(key))


@pytest.mark.parametrize("seed", range(4))
def test_equal_layers_random_configs(seed):
    lin, conv, (x, bias, o) = LC.equal_cases(seed)
    for j, (xl, w, i, o_, act, lr_mul) in enumerate(lin):
        _close(O.equal_linear(xl, w, _g(f"equal_linear_{seed}_{j}_bias"), lr_mul=lr_mul, activation=act is not None),
               _g(f"equal_linear_{seed}_{j}"))
    for j, (xc, w, b, i, o_, k, stride, pad) in enumerate(conv):
        _close(O.equal_conv2d(xc, w, b, stride=stride, padding=pad), _g(f"equal_conv_{seed}_{j}"))
    _close(O.fused_leaky_relu(x, bias), _g(f"fused_lrelu_{seed}"))
    _close(O.pixel_norm(x), _g(f"pixel_norm_{seed}"))


def test_condition_pyramid_equals_bilinear_interpolate():
    """gen.py:309-314 uses F.interpolate(bilinear, align_corners=False); the oracle's closed form (mean of the central 2x2
    of every s x s block) must equal it for every power-of-two factor the generator uses."""
    g = torch.Generator().manual_seed(7)
    cond = torch.rand(2, 6, 256, 256, generator=g, dtype=DT)
    for size in (4, 8, 16, 32, 64, 128, 256):
        ref = torch.nn.functional.interpolate(cond, (size, size), mode="bilinear", align_corners=False)
        _close(O.cond_pyramid_level(cond, size), ref, 1e-12)


def test_minibatch_stddev_and_r1_against_reference_discriminator_tail():
    """disc.py:59-65 (group statistics) through a whole small discriminator in fp64, incl. the R1 penalty's double backward
    (its weight gradient compared on a fixed sample of positions, normalised by the full gradient's largest magnitude)."""
    sd, img, cond = LC.disc_tail_case()
    img2 = img.clone().requires_grad_(True)
    sdo = {k: v.clone() for k, v in sd.items()}
    sdo["final_linear.0.weight"].requires_grad_(True)
    s_o = O.discriminator_forward(img2, cond, sdo, 16)
    pen_o = O.r1_penalty(s_o, img2)
    (g_o,) = torch.autograd.grad(pen_o.mean(), sdo["final_linear.0.weight"])
    _close(s_o, _g("disc_scores"))
    _close(pen_o, _g("disc_r1"))
    g_s = g_o.reshape(-1)[LC.grad_sample_index(g_o.numel())]
    err = float((g_s - _g("disc_r1_grad_sample")).abs().max()) / float(_g("disc_r1_grad_absmax")[0])
    assert err < 1e-9, err
    assert abs(float(g_o.abs().max()) - float(_g("disc_r1_grad_absmax")[0])) <= 1e-9 * float(_g("disc_r1_grad_absmax")[0])
