"""CPU: every write that changes a network's weights is visible to the caches of gif_b200/ops.py.

The prepared-weight cache (``_PrepWeight``) and the staged-operand cache behind it key on a parameter's version counter and
address.  Writes through ``.data`` and raw collectives do not move the counter, so the weight writers of this package
(the EMA ``accumulate``, ``broadcast_module``) must; a parameter rebound with ``p.data = t`` must miss on its address; and a
staged workspace replaced by a larger one must stay allocated, because a captured CUDA graph may still write it."""
import gc
import weakref

import torch


def _net(seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Conv2d(4, 8, 3), torch.nn.ReLU(), torch.nn.Linear(3, 5))


def test_accumulate_bumps_parameter_versions():
    from gif_b200.train_step import accumulate
    m1, m2 = _net(0), _net(1)
    before = [p.detach().clone() for p in m1.parameters()]
    v0 = [p._version for p in m1.parameters()]
    accumulate(m1, m2, decay=0.75)
    for p, v, b, q in zip(m1.parameters(), v0, before, m2.parameters()):
        assert p._version > v
        torch.testing.assert_close(p.detach(), 0.75 * b + 0.25 * q.detach(), rtol=1e-6, atol=1e-7)


def test_broadcast_module_bumps_parameter_versions(monkeypatch):
    from gif_b200 import distributed as D

    def broadcast(t, src):
        t.data.fill_(7.0)             # like the NCCL / gloo collective: an in-place write that no version counter sees

    monkeypatch.setattr(D.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(D.dist, "get_world_size", lambda: 2)
    monkeypatch.setattr(D.dist, "broadcast", broadcast)
    m = _net(0)
    v0 = [p._version for p in m.parameters()]
    D.broadcast_module(m)
    for p, v in zip(m.parameters(), v0):
        assert p._version > v
        assert bool((p.detach() == 7.0).all())


def test_staged_workspace_retires_a_superseded_buffer(monkeypatch):
    from gif_b200 import ops
    monkeypatch.setattr(ops, "_stage_cache", {})
    monkeypatch.setattr(ops, "_ws_retired", [])
    w = torch.zeros(9, 8, 4)
    w._gifb200_prep = (("layer",), 1)                       # what _PrepWeight tags its output with: (prep key, serial)
    cpu = torch.device("cpu")
    ws, fresh = ops._staged_workspace(w, 1000, False, False, 2, (4, 8, 3), cpu)
    assert not fresh and ws.numel() >= 1000
    ws2, fresh = ops._staged_workspace(w, 1000, False, False, 2, (4, 8, 3), cpu)
    assert fresh and ws2 is ws                               # staged from the same serial: reused
    old = weakref.ref(ws)
    del ws, ws2
    ws, fresh = ops._staged_workspace(w, 4000, False, False, 2, (4, 8, 3), cpu)   # a larger batch: more split-K partials
    assert not fresh and ws.numel() >= 4000                  # a new buffer holds no staged operand yet
    gc.collect()
    assert old() is not None, "the superseded staged workspace was freed while a captured graph may still use it"


def test_prep_cache_misses_on_every_weight_change(monkeypatch):
    from gif_b200 import ops
    monkeypatch.setattr(ops, "_prep_cache", {})
    monkeypatch.setattr(ops, "_stage_cache", {})
    g = torch.Generator().manual_seed(0)
    p = torch.nn.Parameter(torch.randn(8, 4, 3, 3, generator=g))

    def prepared():
        out = ops._PrepWeight.apply(p, 0.5)
        want = (p.detach() * 0.5).permute(2, 3, 0, 1).reshape(9, 8, 4)
        assert torch.equal(out, want)
        return out._gifb200_prep[1]

    s0 = prepared()
    assert prepared() == s0                                  # unchanged weights: a hit
    with torch.no_grad():
        p.mul_(2.0)
    s1 = prepared()
    assert s1 != s0
    v = p._version
    p.data = torch.randn(8, 4, 3, 3, generator=g)           # new storage, same version counter
    assert p._version == v
    s2 = prepared()
    assert s2 != s1
    assert prepared() == s2
