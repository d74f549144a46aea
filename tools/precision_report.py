#!/usr/bin/env python
"""Measured deviation from the reference goldens per precision mode (fp32 SIMT / tf32 / bf16x3), network level:
generator 32^2 forward + gradients, generator 256^2 forward, discriminator 64^2 scores + R1 penalty + gradients,
discriminator 256^2 scores.  Prints one JSON line per (mode, quantity); the bars of tests/test_models_gpu.py and of
__graft_entry__.smoke() are set from this table."""
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import golden_util as gu  # noqa: E402
import test_models_gpu as T  # noqa: E402
from gif_b200 import losses, ops  # noqa: E402

cuda = torch.device("cuda:0")


def out(**kw):
    print(json.dumps(kw), flush=True)


for mode in ("fp32", "tf32", "bf16x3"):
    ops.set_precision(mode)
    g = gu.load_golden("generator.npz")
    G, _ = T.make_g(cuda)
    cond = gu.rand_uniform((2, 6, 32, 32), 40).to(cuda).requires_grad_(True)
    idx = gu.randint(100, (2,), 41).to(cuda)
    img = G(cond, step=3, input_indices=idx)[0]
    gy = gu.randn(tuple(img.shape), 42).to(cuda)
    named = dict(G.named_parameters())
    grads = torch.autograd.grad((img * gy).sum(), [cond] + [named[n] for n in T.G_PNAMES])
    out(mode=mode, what="G32 forward max-rel", err=gu.rel_err(img.detach().cpu().numpy(), g["s3_img"]))
    out(mode=mode, what="G32 grad cond L2 vs f64", err=T.l2rel(grads[0].cpu().numpy(), g["s3_gcond_f64"]))
    out(mode=mode, what="G32 param grads L2 vs f64 (max over watched)",
        err=max(T.l2rel(gu.sample(gr, 2048, 2)[0], g["s3_g64_" + n]) for n, gr in zip(T.G_PNAMES, grads[1:])))
    with torch.no_grad():
        img = G(gu.rand_uniform((2, 6, 256, 256), 44).to(cuda), step=6, input_indices=gu.randint(100, (2,), 45).to(cuda))[0]
    s, tot = gu.sample(img, 8192, 3)
    out(mode=mode, what="G256 forward max-rel (sampled)", err=float(np.abs(s - g["s6_sample"]).max() / float(g["s6_absmax"])))
    del G
    g = gu.load_golden("discriminator.npz")
    D, _ = T.make_d(cuda, 64, 2)
    img = gu.rand_uniform((8, 3, 64, 64), 50).to(cuda).requires_grad_(True)
    cond = gu.rand_uniform((8, 6, 64, 64), 51).to(cuda).requires_grad_(True)
    scores, _ = D([img], condition=cond)
    pen = losses.grad_penalty_loss([img], scores, step=None)
    loss = F.softplus(-scores).mean() + pen.mean()
    named = dict(D.named_parameters())
    grads = torch.autograd.grad(loss, [img, cond] + [named[n] for n in T.D_PNAMES])
    out(mode=mode, what="D64 scores max-rel", err=gu.rel_err(scores.detach().cpu().numpy(), g["d64_scores"]))
    out(mode=mode, what="D64 R1 penalty max-rel", err=gu.rel_err(pen.detach().cpu().numpy(), g["d64_r1"]))
    out(mode=mode, what="D64 grad img L2 vs f64", err=T.l2rel(grads[0].cpu().numpy(), g["d64_gimg_f64"]),
        reference_fp32_floor=float(g["d64_gimg_ref32_l2err"]))
    out(mode=mode, what="D64 grad cond L2 vs f64", err=T.l2rel(grads[1].cpu().numpy(), g["d64_gcond_f64"]))
    out(mode=mode, what="D64 param grads (softplus + R1) L2 vs f64 (max over watched)",
        err=max(T.l2rel(gu.sample(gr, 2048, 4)[0], g["d64_g64_" + n]) for n, gr in zip(T.D_PNAMES, grads[2:])))
    del D
    D, _ = T.make_d(cuda, 256, 3)
    with torch.no_grad():
        scores, _ = D([gu.rand_uniform((4, 3, 256, 256), 52).to(cuda)], condition=gu.rand_uniform((4, 6, 256, 256), 53).to(cuda))
    out(mode=mode, what="D256 scores max-rel", err=gu.rel_err(scores.cpu().numpy(), g["d256_scores"]))
    del D
    torch.cuda.empty_cache()
ops.set_precision("tf32")
