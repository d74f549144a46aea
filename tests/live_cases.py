"""Seeded inputs of the comparisons with the unmodified reference (tests/test_oracle_vs_reference_live.py, test_fid_cpu.py,
test_checkpoint.py).  oracle/make_live_golden.py ran the reference on exactly these inputs and stored its outputs in
tests/golden/reference_live.npz; the tests regenerate the inputs and compare this repo's code with those outputs."""
import numpy as np
import torch

DT = torch.float64
CHECKPOINT_KW = dict(embedding_vocab_size=32, rendered_flame_ascondition=True, normal_maps_as_cond=True, core_tensor_res=4,
                     n_mlp=8)
GRAD_SAMPLE = 8192


def upfirdn_cases(seed):
    """[(x, kernel, up, down, pad)] -- random up / down / pad / sizes, the empty-output draws skipped."""
    g = torch.Generator().manual_seed(seed)
    cases = []
    for _ in range(6):
        up, down = int(torch.randint(1, 3, (1,), generator=g)), int(torch.randint(1, 3, (1,), generator=g))
        p0, p1 = int(torch.randint(-1, 4, (1,), generator=g)), int(torch.randint(0, 4, (1,), generator=g))
        h, w = int(torch.randint(5, 14, (1,), generator=g)), int(torch.randint(5, 14, (1,), generator=g))
        kh = int(torch.randint(2, 5, (1,), generator=g))
        k = torch.randn(kh, kh, generator=g, dtype=DT)
        x = torch.randn(2, 3, h, w, generator=g, dtype=DT)
        if (h * up + p0 + p1 - kh) // down + 1 <= 0 or (w * up + p0 + p1 - kh) // down + 1 <= 0:
            continue
        cases.append((x, k, up, down, (p0, p1)))
    return cases


def modconv_case(seed, upsample, demod):
    """ModulatedConv2d(ci, co, k, style_dim=7) parameters (reference shapes) and inputs."""
    g = torch.Generator().manual_seed(100 + seed)
    ci, co = int(torch.randint(2, 9, (1,), generator=g)), int(torch.randint(2, 9, (1,), generator=g))
    k = 3 if upsample or seed % 2 == 0 else 1
    r, b, sdim = int(torch.randint(3, 8, (1,), generator=g)), int(torch.randint(1, 4, (1,), generator=g)), 7
    c = dict(ci=ci, co=co, k=k, sdim=sdim)
    c["weight"] = torch.randn((1, co, ci, k, k), generator=g, dtype=DT)
    c["mod_weight"] = torch.randn((ci, sdim), generator=g, dtype=DT)
    c["mod_bias"] = torch.randn((ci,), generator=g, dtype=DT)
    c["x"] = torch.randn(b, ci, r, r, generator=g, dtype=DT)
    c["s"] = torch.randn(b, sdim, generator=g, dtype=DT)
    return c


def equal_cases(seed):
    """EqualLinear cases [(x, w, i, o, activation, lr_mul)], EqualConv2d cases [(x, w, b, i, o, k, stride, pad)] and the
    FusedLeakyReLU / PixelNorm input (x, bias, o)."""
    g = torch.Generator().manual_seed(200 + seed)
    i, o = int(torch.randint(2, 20, (1,), generator=g)), int(torch.randint(2, 20, (1,), generator=g))
    lin = []
    for act, lr_mul in ((None, 1.0), ("fused_lrelu", 0.01), (None, 0.5)):
        w = torch.randn(o, i, generator=g, dtype=DT) / lr_mul
        lin.append((torch.randn(5, i, generator=g, dtype=DT), w, i, o, act, lr_mul))
    conv = []
    for k, stride, pad, r in ((1, 1, 0, 6), (3, 1, 1, 6), (3, 2, 0, 9), (1, 2, 0, 7)):
        w = torch.randn((o, i, k, k), generator=g, dtype=DT)
        b = torch.randn(o, generator=g, dtype=DT)
        conv.append((torch.randn(2, i, r, r, generator=g, dtype=DT), w, b, i, o, k, stride, pad))
    bias = torch.randn((1, o, 1, 1), generator=g, dtype=DT)
    x = torch.randn(3, o, 4, 5, generator=g, dtype=DT)
    return lin, conv, (x, bias, o)


def disc_tail_case():
    """Discriminator(16, 9 channels) state_dict, image and condition (fp64)."""
    import golden_util as gu
    sd = {k: v.double() for k, v in gu.seeded_state_dict(gu.d_shapes(16), 31).items()}
    return sd, gu.rand_uniform((8, 3, 16, 16), 32).double(), gu.rand_uniform((8, 6, 16, 16), 33).double()


def grad_sample_index(n):
    """Positions of the stored sample of a large reference gradient (the same on every run)."""
    return torch.randperm(n, generator=torch.Generator().manual_seed(0))[:GRAD_SAMPLE].sort().values


def fid_case():
    rng = np.random.default_rng(5)
    a, b = rng.normal(size=(400, 96)), rng.normal(size=(400, 96)) @ rng.normal(size=(96, 96)) * 0.2
    return a.mean(0), np.cov(a, rowvar=False), b.mean(0), np.cov(b, rowvar=False)
