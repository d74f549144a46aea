"""GPU: the per-tensor operand marks that tensor-core convolutions trust, checked on every operand of a whole training
iteration (R1 and path-length terms included) and of an FID Inception forward.

* ``_gifb200_tf32``: a tensor marked tf32-representable at its current version has the low 13 mantissa bits zero
  (the wgmma tf32 path then skips its rounding pass and truncates).
* ``_gifb200_planes``: valid bf16x3 planes of a tensor whose fp32 values were written are bitwise torch's round-to-nearest
  split of those values: hi = bf16(x), lo = bf16(x - hi).

A gradient that exists only as planes (a carrier: the fused activation backward writes the planes and leaves the fp32
tensor unwritten) has no values to compare, so the bf16x3 iteration is also run with carriers disabled
(``ops._x3_backward_on_planes`` returning False): every gradient must be bitwise the same."""
import pytest
import torch

import golden_util as gu

pytestmark = pytest.mark.gpu


def _check(t, mode, counts):
    from gif_b200 import ops
    if t is None:
        return
    if mode == "tf32" and ops._is_tf32(t):
        assert not bool((t.detach().view(torch.int32) & 0x1FFF).any()), f"tensor {tuple(t.shape)} marked tf32 is not"
        counts["tf32"] += 1
    c = getattr(t, "_gifb200_planes", None)
    if mode == "bf16x3" and c is not None and c[0] == t._version:
        v = t.detach()
        hi = v.bfloat16()
        lo = (v - hi.float()).bfloat16()
        assert torch.equal(c[1][0].view(torch.int16), hi.view(torch.int16)), f"hi plane of {tuple(t.shape)}"
        assert torch.equal(c[1][1].view(torch.int16), lo.view(torch.int16)), f"lo plane of {tuple(t.shape)}"
        counts["planes"] += 1


def _watch(monkeypatch, mode):
    """Wraps the three convolution entry points: operands are checked before each call, and again after it (the call may
    have rounded or split them and cached the result on the tensor)."""
    from gif_b200 import ops
    counts = {"tf32": 0, "planes": 0, "calls": 0}
    conv_raw, wgrad_raw, conv2d_ex = ops._conv_raw, ops._wgrad_raw, ops.conv2d_ex

    def conv(x, w, *a, **kw):
        _check(x, mode, counts)
        y, x_used = conv_raw(x, w, *a, **kw)
        _check(x, mode, counts)
        _check(x_used, mode, counts)
        counts["calls"] += 1
        return y, x_used

    def wgrad(x, gy, *a, **kw):
        _check(x, mode, counts)
        _check(gy, mode, counts)
        gw = wgrad_raw(x, gy, *a, **kw)
        _check(x, mode, counts)
        _check(gy, mode, counts)
        counts["calls"] += 1
        return gw

    def ex(x, w, *a, **kw):
        _check(x, mode, counts)
        y = conv2d_ex(x, w, *a, **kw)
        _check(x.contiguous(), mode, counts)
        counts["calls"] += 1
        return y

    monkeypatch.setattr(ops, "_conv_raw", conv)
    monkeypatch.setattr(ops, "_wgrad_raw", wgrad)
    monkeypatch.setattr(ops, "conv2d_ex", ex)
    return counts


def _iteration(cuda):
    """One eager GifTrainer iteration with the R1 penalty and the path-length term; returns losses and every gradient."""
    from gif_b200.train_step import GifTrainer
    tr = GifTrainer(cuda, 32, vocab=16, r1_every=1, ppl=True, seed=4)
    b = 4
    batch = (gu.rand_uniform((b, 3, 32, 32), 80).to(cuda), gu.rand_uniform((b, 6, 32, 32), 81).to(cuda),
             gu.randint(16, (b,), 82).to(cuda))
    losses = [float(v) for v in tr.train_iteration(*batch)]
    grads = [p.grad.clone() for m in (tr.generator, tr.discriminator) for p in m.parameters() if p.grad is not None]
    return losses, grads


def _inception(cuda):
    from gif_b200.inception import InceptionV3
    from oracle import inception_oracle as IO
    net = InceptionV3([0, 1, 2, 3], weights=IO.golden_state_dict(gu.load_golden("fid_inception.npz"))).to(cuda)
    with torch.no_grad():
        net(torch.rand(2, 3, 96, 96, generator=torch.Generator().manual_seed(83)).to(cuda))


@pytest.mark.parametrize("mode", ["tf32", "bf16x3"])
def test_operand_marks_hold_over_an_iteration_and_inception(cuda, monkeypatch, mode):
    from gif_b200 import ops
    old = ops.get_precision()
    ops.set_precision(mode)
    try:
        if mode == "bf16x3":       # no carriers: every tensor holding planes also holds its fp32 values
            monkeypatch.setattr(ops, "_x3_backward_on_planes", lambda *a: False)
        counts = _watch(monkeypatch, mode)
        _iteration(cuda)
        _inception(cuda)
    finally:
        ops.set_precision(old)
    assert counts["calls"] > 100
    assert counts["tf32" if mode == "tf32" else "planes"] > 100, counts


def test_planes_carriers_change_no_gradient(cuda, monkeypatch):
    """The carrier path (planes written by the fused activation backward, fp32 never written) against the path that writes
    the fp32 gradient and splits it: same losses, bitwise the same gradients."""
    from gif_b200 import ops
    old = ops.get_precision()
    ops.set_precision("bf16x3")
    try:
        carriers = [0]
        real = ops._x3_backward_on_planes

        def counting(*a):
            r = real(*a)
            carriers[0] += int(r)
            return r
        monkeypatch.setattr(ops, "_x3_backward_on_planes", counting)
        l_a, g_a = _iteration(cuda)
        assert carriers[0] > 0, "no carrier was produced: the comparison would be vacuous"
        monkeypatch.setattr(ops, "_x3_backward_on_planes", lambda *a: False)
        l_b, g_b = _iteration(cuda)
    finally:
        ops.set_precision(old)
    assert l_a == l_b
    assert len(g_a) == len(g_b)
    for i, (a, b) in enumerate(zip(g_a, g_b)):
        assert torch.equal(a, b), f"gradient {i}: max diff {float((a - b).abs().max()):.3e}"
