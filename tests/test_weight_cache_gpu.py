"""GPU: a network evaluated after its weights changed uses the new weights, whatever changed them.

Training-mode layers keep their prepared weights (``ops._PrepWeight``) and the staged tensor-core operand of those weights
(``ops._staged_workspace``) between calls, keyed on the parameters' version counters and addresses.  Each test evaluates a
network, changes its weights in one of the ways a training or sampling loop does, evaluates again, and requires the
second output to (1) differ from the first, (2) be bitwise equal to the same evaluation with both caches off (the prep and
staging arithmetic is the same, so the bits must match) and (3) agree with the float64 oracle on the changed weights
within the forward bar of tests/test_models_gpu.py.  The CUDA-graph test does the same between replays of
``GifTrainer``'s captured iteration, whose parameter writes run no Python."""
import copy

import pytest
import torch

import golden_util as gu
from oracle import stylegan2_oracle as O

pytestmark = pytest.mark.gpu

FWD_BAR = {"fp32": 5e-5, "tf32": 3e-3, "bf16x3": 2e-4}      # tests/test_models_gpu.py, G 32^2 and D forward


@pytest.fixture
def precision(request):
    from gif_b200 import ops
    old = ops.get_precision()
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(old)


@pytest.fixture(scope="module")
def nets(cuda):
    from gif_b200.model.stg2_discriminator import Discriminator
    from gif_b200.model.stg2_generator import StyledGenerator
    G = StyledGenerator(embedding_vocab_size=100, rendered_flame_ascondition=True, normal_maps_as_cond=True,
                        core_tensor_res=4, n_mlp=8)
    G.load_state_dict(gu.seeded_state_dict(gu.g_shapes(100), 1))
    D = Discriminator(32, num_color_chnls=9)
    D.load_state_dict(gu.seeded_state_dict(gu.d_shapes(32), 2))
    return {"G": G.to(cuda), "D": D.to(cuda)}


class _Net:
    """One module under test, its seeded inputs at batch ``b``, and its float64 oracle."""

    def __init__(self, which, module, cuda, b=None):
        self.which, self.m = which, module
        b = b or (2 if which == "G" else 4)
        self.cond = gu.rand_uniform((b, 6, 32, 32), 40 + b)
        if which == "G":
            self.idx = gu.randint(100, (b,), 41 + b)
            self.args = (self.cond.to(cuda), self.idx.to(cuda))
        else:
            self.img = gu.rand_uniform((b, 3, 32, 32), 42 + b)
            self.args = (self.img.to(cuda), self.cond.to(cuda))

    def __call__(self, module=None):
        m = self.m if module is None else module
        if self.which == "G":
            return m(self.args[0], step=3, input_indices=self.args[1])[0]
        return m([self.args[0]], condition=self.args[1])[0]

    def eval(self, module=None, cached=True):
        from gif_b200 import ops
        with torch.no_grad(), pytest.MonkeyPatch.context() as mp:
            if not cached:
                mp.setattr(ops, "_NO_WEIGHT_CACHE", True)
            return self(module).clone()

    def oracle(self, module):
        sd = {k: v.detach().cpu().double() for k, v in module.state_dict().items()}
        if self.which == "G":
            return O.generator_forward(self.cond.double(), self.idx, sd, step=3)
        return O.discriminator_forward(self.img.double(), self.cond.double(), sd, 32)


def _noise_like(m, seed, scale):
    g = torch.Generator().manual_seed(seed)
    return [scale * torch.randn(p.shape, generator=g).to(p.device) for p in m.parameters()]


def _adam_step(net, opt_cls):
    m = net.m
    opt = opt_cls([p for p in m.parameters() if p.requires_grad], lr=1e-2, betas=(0.0, 0.99))
    out = net()
    (out * gu.randn(tuple(out.shape), 7).to(out.device)).sum().backward()
    opt.step()
    return m


def _fused_adam(net):
    from gif_b200.optim import FusedAdam
    return _adam_step(net, FusedAdam)


def _torch_adam(net):
    return _adam_step(net, torch.optim.Adam)


def _load_state_dict(net):
    params = dict(net.m.named_parameters())
    sd = {k: v + 0.01 * gu.randn(tuple(v.shape), 8).to(v.device) if k in params else v
          for k, v in net.m.state_dict().items()}
    net.m.load_state_dict(sd)
    return net.m


def _inplace_no_grad(net):
    with torch.no_grad():
        for p, n in zip(net.m.parameters(), _noise_like(net.m, 9, 0.01)):
            p.add_(n)
    return net.m


def _rebind_data(net):
    for p, n in zip(net.m.parameters(), _noise_like(net.m, 10, 0.01)):
        p.data = p.data + n                       # new storage; the version counter does not move
    return net.m


def _ema(write):
    """An eval-mode copy (the EMA generator of train.py / GifTrainer) evaluated, then moved towards the trained network."""
    def mutate(net):
        ema = copy.deepcopy(net.m).train(False)
        net.first = net.eval(ema)
        _inplace_no_grad(net)
        write(ema, net.m, 0.5)
        return ema
    return mutate


def _reference_accumulate(m1, m2, decay):
    """my_utils/generic_utils.py:63-76, which train.py:250 calls: an in-place update through ``.data``."""
    par1, par2 = dict(m1.named_parameters()), dict(m2.named_parameters())
    for k in par1:
        par1[k].data.mul_(decay).add_(par2[k].data, alpha=1 - decay)


def _accumulate(m1, m2, decay):
    from gif_b200.train_step import accumulate
    accumulate(m1, m2, decay)


MUTATIONS = {"fused_adam": _fused_adam, "torch_adam": _torch_adam, "load_state_dict": _load_state_dict,
             "inplace_no_grad": _inplace_no_grad, "rebind_data": _rebind_data, "ema_accumulate": _ema(_accumulate),
             "ema_reference_data": _ema(_reference_accumulate)}


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16x3"], indirect=True)
@pytest.mark.parametrize("which", ["G", "D"])
@pytest.mark.parametrize("how", list(MUTATIONS))
def test_output_follows_the_weights(cuda, nets, precision, which, how):
    net = _Net(which, copy.deepcopy(nets[which]), cuda)
    net.first = net.eval()
    target = MUTATIONS[how](net)
    first = net.first
    second = net.eval(target)
    uncached = net.eval(target, cached=False)
    assert torch.equal(second, uncached), \
        f"stale cached weights: max |cached - uncached| = {float((second - uncached).abs().max()):.3e}"
    assert not torch.equal(second, first), "the weight change did not reach the output: the check would be vacuous"
    err = gu.rel_err(second.cpu().numpy(), net.oracle(target).numpy())
    assert err < FWD_BAR[precision], f"{which} after {how} [{precision}]: rel err vs float64 oracle {err:.2e}"


def _spy_staging(monkeypatch, log, batch):
    from gif_b200 import ops
    real = ops._staged_workspace

    def spy(w, nws, flip, transposed, impl, shape_key, device):
        tag = getattr(w, "_gifb200_prep", None)
        key = None if tag is None else (tag[0], bool(flip), bool(transposed), impl, shape_key)
        ent = ops._stage_cache.get(key) if key is not None else None
        prior = None if ent is None else ent[1].numel()
        ws, fresh = real(w, nws, flip, transposed, impl, shape_key, device)
        if key is not None and nws > 0:
            log.append(dict(key=key, batch=batch[0], nws=nws, grew=prior is not None and prior < nws, fresh=fresh))
        return ws, fresh
    monkeypatch.setattr(ops, "_staged_workspace", spy)


def _check_staging_coverage(log):
    by_key = {}
    for e in log:
        by_key.setdefault(e["key"], []).append(e)
    assert any(e["grew"] for e in log), "no staged workspace grew"
    assert any(e["fresh"] for e in log) and any(not e["fresh"] for e in log)
    assert {e["key"][3] for e in log} >= {0, 3}, "tf32 (impl 0) and bf16x3 (impl 3) staging both exercised"
    # split-K partials scale with the batch; a non-split layer's workspace is the staged operand alone
    assert any(len({e["nws"] for e in es}) > 1 for es in by_key.values()), "no split-K layer"
    assert any(len({e["batch"] for e in es}) > 1 and len({e["nws"] for e in es}) == 1 for es in by_key.values()), \
        "no non-split layer"


@pytest.mark.parametrize("which", ["G", "D"])
def test_staged_operands_across_modes_and_batches(cuda, nets, monkeypatch, which):
    """One set of weights, evaluated in alternating precision modes and batch sizes: the staged operand of a layer is reused,
    restaged (new impl or new weights), and grown (split-K partials at a larger batch), and never read stale."""
    from gif_b200 import ops
    m = copy.deepcopy(nets[which])
    batch, log = [0], []
    _spy_staging(monkeypatch, log, batch)
    b0 = 2 if which == "G" else 4
    seq = [("tf32", b0), ("bf16x3", b0), ("tf32", b0), ("tf32", 4 * b0), ("bf16x3", 4 * b0), ("fp32", b0),
           ("bf16x3", b0), ("bf16x3", 4 * b0), ("tf32", 2 * b0), ("bf16x3", 2 * b0)]
    old = ops.get_precision()
    try:
        for mode, b in seq:
            ops.set_precision(mode)
            batch[0] = b
            net = _Net(which, m, cuda, b)
            y, y0 = net.eval(), net.eval(cached=False)
            assert torch.equal(y, y0), (mode, b, float((y - y0).abs().max()))
    finally:
        ops.set_precision(old)
    _check_staging_coverage(log)


def _batch(seed, b, dev):
    return (gu.rand_uniform((b, 3, 32, 32), seed).to(dev), gu.rand_uniform((b, 6, 32, 32), seed + 1).to(dev),
            gu.randint(16, (b,), seed + 2).to(dev))


def _evaluate_all(tr, b, dev):
    """G, D and the EMA generator under no_grad with the caches on, each bitwise equal to its uncached twin."""
    from gif_b200 import ops
    real, cond, idx = _batch(1000 + b, b, dev)
    nets = [("G", lambda: tr.generator(cond, step=3, input_indices=idx)[0]),
            ("g_running", lambda: tr.g_running(cond, step=3, input_indices=idx)[0]),
            ("D", lambda: tr.discriminator([real], condition=cond)[0])]
    for name, fn in nets:
        with torch.no_grad():
            y = fn().clone()
            with pytest.MonkeyPatch.context() as mp:
                mp.setattr(ops, "_NO_WEIGHT_CACHE", True)
                y0 = fn().clone()
        assert torch.equal(y, y0), f"{name} at batch {b}: stale cached weights, max diff {float((y - y0).abs().max()):.3e}"


def _run_trainer(cuda, evaluate, growth):
    from gif_b200.train_step import GifTrainer
    tr = GifTrainer(cuda, 32, vocab=16, r1_every=2, ppl=False, seed=3)
    losses = []

    def iterate(n):
        for _ in range(n):
            losses.append(tuple(float(v) for v in tr.train_iteration(*_batch(10 * len(losses), 4, cuda))))

    iterate(2)
    tr.capture(4, 32)
    iterate(3)
    for _ in range(2):
        if evaluate:
            _evaluate_all(tr, 4, cuda)
        iterate(2)
    if growth:
        if evaluate:
            _evaluate_all(tr, 16, cuda)     # larger split-K partials: the staged workspaces of G and D grow
        iterate(2)
    return losses


@pytest.mark.parametrize("precision", ["tf32", "bf16x3"], indirect=True)
@pytest.mark.parametrize("scenario", ["steady", "growth"])
def test_eager_evaluation_between_graph_replays(cuda, precision, scenario, monkeypatch):
    """Eager evaluations of G, D and the EMA generator between CUDA-graph replays see the weights the replays wrote, and
    (with a batch that grows the staged workspaces) do not disturb the captured iteration: the losses are bitwise those of
    a twin trainer that never evaluated."""
    log, batch = [], [0]
    _spy_staging(monkeypatch, log, batch)
    got = _run_trainer(cuda, True, scenario == "growth")
    if scenario == "growth":
        assert any(e["grew"] for e in log), "the batch-16 evaluation did not grow a staged workspace"
    want = _run_trainer(cuda, False, scenario == "growth")
    assert got == want
