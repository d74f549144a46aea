"""CPU: checkpoint round trip in the format of the unmodified reference (train.py:255-262 / 389-395).  The reference networks'
state_dict keys, shapes and parameter order are stored in tests/golden/reference_live.npz (oracle/make_live_golden.py).
A checkpoint laid out the way train.py writes it (DataParallel ``module.`` keys + torch Adam states indexed by the
reference's parameter order) loads into the gif_b200 modules with strict=True, and what gif_b200 writes has the reference's
layout, so the reference modules read it back."""
import io

import pytest
import torch

import golden_util as gu
import live_cases as LC


def _schema(tag):
    g = gu.load_golden("reference_live.npz")
    shapes = [tuple(int(v) for v in s.split(",")) if s else () for s in g[f"schema_{tag}_shapes"]]
    return list(g[f"schema_{tag}_keys"]), shapes, list(g[f"schema_{tag}_param_order"])


def _seeded(keys, shapes, seed, net):
    """Seeded values for every key; state_dict entries that alias one tensor (the identity embedding) end up equal, as in
    a state_dict the reference writes."""
    gen = torch.Generator().manual_seed(seed)
    net.load_state_dict({k: torch.randn(s, generator=gen) for k, s in zip(keys, shapes)}, strict=True)
    return {k: v.clone() for k, v in net.state_dict().items()}


def _adam(params, lr):
    opt = torch.optim.Adam(params, lr=lr, betas=(0.0, 0.99))
    g = torch.Generator().manual_seed(1)
    for p in params:
        p.grad = torch.randn(p.shape, generator=g) * 0.01
    opt.step()
    return opt


def test_reference_checkpoint_round_trip():
    from gif_b200 import checkpoint
    from gif_b200.model.stg2_discriminator import Discriminator
    from gif_b200.model.stg2_generator import StyledGenerator
    gk, gs, gorder = _schema("g")
    dk, ds, dorder = _schema("d")
    G, Gr = StyledGenerator(**LC.CHECKPOINT_KW), StyledGenerator(**LC.CHECKPOINT_KW)
    D = Discriminator(64, num_color_chnls=9, channel_multiplier=2)
    # the reference's layout: keys in order, shapes, parameter order
    for net, keys, shapes, order in ((G, gk, gs, gorder), (D, dk, ds, dorder)):
        sd = net.state_dict()
        assert list(sd) == keys
        assert [tuple(v.shape) for v in sd.values()] == shapes
        names = {id(p): n for n, p in net.named_parameters()}
        assert [names[id(p)] for p in net.parameters()] == order
    # what train.py:257-262 saves (nn.DataParallel adds the `module.` prefix); Adam state for D only (G is the same path)
    sd_g, sd_gr = _seeded(gk, gs, 2, StyledGenerator(**LC.CHECKPOINT_KW)), _seeded(gk, gs, 3, StyledGenerator(**LC.CHECKPOINT_KW))
    sd_d = _seeded(dk, ds, 4, Discriminator(64, num_color_chnls=9, channel_multiplier=2))
    rd_params = [torch.nn.Parameter(sd_d[n].clone()) for n in dorder]
    rdo = _adam(rd_params, 2e-3)
    rgo = torch.optim.Adam([torch.nn.Parameter(sd_g[n].clone()) for n in gorder], lr=1e-3, betas=(0.0, 0.99))
    pre = checkpoint.add_dataparallel_prefix
    ck = {"generator_running": pre(sd_gr), "generator": pre(sd_g), "g_optimizer": rgo.state_dict(),
          "discriminator_flm": pre(sd_d), "d_optimizer_flm": rdo.state_dict()}
    buf = io.BytesIO()
    torch.save({"discriminator_flm": ck["discriminator_flm"], "d_optimizer_flm": ck["d_optimizer_flm"]}, buf)   # file round trip
    buf.seek(0)
    ck.update(torch.load(buf, weights_only=True))
    go = torch.optim.Adam(G.parameters(), lr=5e-4, betas=(0.0, 0.9))
    do = torch.optim.Adam(D.parameters(), lr=5e-4, betas=(0.0, 0.9))
    checkpoint.load_reference_checkpoint(ck, G, Gr, D, go, do, strict=True)
    for ours, want in ((G, sd_g), (Gr, sd_gr), (D, sd_d)):
        so = ours.state_dict()
        assert all(torch.equal(so[k], want[k]) for k in want)
    # Adam moments follow the parameter ORDER: identical order => identical per-parameter state
    for p, rp in zip(D.parameters(), rd_params):
        assert torch.equal(do.state[p]["exp_avg_sq"], rdo.state[rp]["exp_avg_sq"])
    assert do.param_groups[0]["lr"] == 5e-4 and len(go.state) == 0     # this optimiser's hyper-parameters are kept
    # and back: what gif_b200 writes has the reference's keys and shapes (train.py:389-395 loads it into its modules)
    out = checkpoint.reference_checkpoint_dict(G, Gr, D, go, do)
    for key, keys, shapes in (("generator", gk, gs), ("generator_running", gk, gs), ("discriminator_flm", dk, ds)):
        assert list(out[key]) == ["module." + k for k in keys]
        assert [tuple(v.shape) for v in out[key].values()] == shapes
    assert all(torch.equal(out["generator"]["module." + k], sd_g[k]) for k in gk)
    ro = torch.optim.Adam([torch.nn.Parameter(sd_d[n].clone()) for n in dorder], lr=1e-3, betas=(0.0, 0.99))
    ro.load_state_dict(out["d_optimizer_flm"])
    assert checkpoint.strip_dataparallel_prefix({"module.a": 1, "b": 2}) == {"a": 1, "b": 2}
    with pytest.raises(KeyError):
        checkpoint.load_reference_checkpoint({"generator": {}}, g_running=Gr)
