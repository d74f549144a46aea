"""TEST INFRASTRUCTURE ONLY -- writes ``tests/golden/highres.npz``: the UNMODIFIED reference modules (imported from the
reference tree through ``oracle/ref_import.py``) evaluated in float64 on the CPU at 512^2, and the agreement of the in-repo
oracle with them at that size, in ``tests/golden/HIGHRES_ORACLE_VS_REFERENCE.txt``.

  * StyledGenerator at step 7 (512^2), batch 2, with a 512^2 condition and with a 256^2 condition (the reference's
    F.interpolate then upsamples the 512^2 level): image and first derivatives w.r.t. the condition and sampled weights;
  * Discriminator(512, 9 ch), batch 4: scores, R1 penalty, gradients of softplus + R1 w.r.t. sampled weights, and the
    reference's own float32 error of the scores and of R1 (the floor the CUDA path is compared with).

The sampled weights include the narrow (32- / 64-channel) layers.  Tensors are stored as seeded samples
(``golden_util.sample``).  The oracle's condition pyramid reduces only; for the upsampling case it is evaluated with
F.interpolate at every level, which is what the reference does, and the agreement recorded here pins that.

Run where the reference tree exists (a few minutes on 8 cores):   python tools/make_highres_golden.py
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import golden_util as gu  # noqa: E402
from oracle import ref_import  # noqa: E402
from oracle import stylegan2_oracle as O  # noqa: E402

VOCAB = 16
G_NAMES = ["generator.progression.7.st_cv1.conv.weight", "generator.progression.7.st_cv2.conv.weight",
           "generator.progression.7.st_cv2.noise.noise_conv.4.weight", "generator.progression.5.st_cv2.conv.weight"]
D_NAMES = ["convs.0.0.weight", "convs.1.conv1.0.weight", "convs.1.conv2.1.weight", "convs.1.skip.1.weight",
           "final_conv.0.weight"]
report = []


def check(name, a, b, tol):
    e = gu.rel_err(a.detach().double().numpy(), b.detach().double().numpy())
    report.append((name, e))
    assert e < tol, f"oracle != reference for {name}: rel err {e:.3e} (tol {tol})"


def bilinear(c, size):
    return F.interpolate(c, size=(size, size), mode="bilinear", align_corners=False)


def generator(R, out):
    with ref_import.quiet():
        G = R.gen.StyledGenerator(embedding_vocab_size=VOCAB, rendered_flame_ascondition=True, normal_maps_as_cond=True,
                                  core_tensor_res=4, n_mlp=8)
    sd = gu.seeded_state_dict(gu.g_shapes(VOCAB), 11)
    G.load_state_dict(sd)
    G = G.double()
    named = dict(G.named_parameters())
    idx = gu.randint(VOCAB, (2,), 13)
    gy = gu.randn((2, 3, 512, 512), 14).double()
    for cres in (512, 256):
        cond = gu.rand_uniform((2, 6, cres, cres), 12).double().requires_grad_(True)
        img = G(cond, step=7, input_indices=idx)[0]
        grads = torch.autograd.grad((img * gy).sum(), [cond] + [named[n] for n in G_NAMES])
        sd_q = {k: v.double().requires_grad_(k in G_NAMES) for k, v in sd.items()}
        cond_q = cond.detach().clone().requires_grad_(True)
        pyramid = O.cond_pyramid_level
        O.cond_pyramid_level = bilinear if cres < 512 else pyramid
        try:
            img_q = O.generator_forward(cond_q, idx, sd_q, step=7)
        finally:
            O.cond_pyramid_level = pyramid
        g_q = torch.autograd.grad((img_q * gy).sum(), [cond_q] + [sd_q[n] for n in G_NAMES])
        tag = f"g512_c{cres}"
        check(f"G[step7, cond {cres}].img fp64", img_q, img, 1e-10)
        for n, a, b in zip(["cond"] + G_NAMES, g_q, grads):
            check(f"G[step7, cond {cres}].g[{n}] fp64", a, b, 1e-9)
        s, tot = gu.sample(img, 8192, 5)
        out[f"{tag}_img"], out[f"{tag}_img_sum"], out[f"{tag}_img_absmax"] = s, tot, float(img.abs().max())
        for n, g in zip(["cond"] + G_NAMES, grads):
            out[f"{tag}_g_{n}"] = gu.sample(g, 4096, 6)[0]
        print(tag, "done", flush=True)


def discriminator(R, out):
    with ref_import.quiet():
        D = R.disc.Discriminator(512, num_color_chnls=9)
    sd = gu.seeded_state_dict(gu.d_shapes(512), 21)
    D.load_state_dict(sd)
    img = gu.rand_uniform((4, 3, 512, 512), 22)
    cond = gu.rand_uniform((4, 6, 512, 512), 23)
    # the reference in float32: its own error is the floor of the score / R1 comparisons
    x32 = img.clone().requires_grad_(True)
    s32, _ = D([x32], condition=cond)
    p32 = R.losses.grad_penalty_loss([x32], s32, step=None)
    D = D.double()
    named = dict(D.named_parameters())
    x = img.double().requires_grad_(True)
    scores, _ = D([x], condition=cond.double())
    pen = R.losses.grad_penalty_loss([x], scores, step=None)
    grads = torch.autograd.grad(F.softplus(-scores).mean() + pen.mean(), [named[n] for n in D_NAMES])
    sd_q = {k: v.double().requires_grad_(k in D_NAMES) for k, v in sd.items()}
    x_q = img.double().requires_grad_(True)
    s_q = O.discriminator_forward(x_q, cond.double(), sd_q, 512)
    p_q = O.r1_penalty(s_q, x_q)
    g_q = torch.autograd.grad(F.softplus(-s_q).mean() + p_q.mean(), [sd_q[n] for n in D_NAMES])
    check("D[512].scores fp64", s_q, scores, 1e-10)
    check("D[512].r1 fp64", p_q, pen, 1e-10)
    for n, a, b in zip(D_NAMES, g_q, grads):
        check(f"D[512].g[{n}] fp64", a, b, 1e-9)
    out["d512_scores"] = scores.detach().numpy()
    out["d512_r1"] = pen.detach().numpy()
    out["d512_scores_ref32_err"] = gu.rel_err(s32.detach().double().numpy(), scores.detach().numpy())
    out["d512_r1_ref32_err"] = gu.rel_err(p32.detach().double().numpy(), pen.detach().numpy())
    for n, g in zip(D_NAMES, grads):
        out[f"d512_g_{n}"] = gu.sample(g, 4096, 7)[0]
    print("d512 done", flush=True)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count() or 8)
    R = ref_import.load()
    out = {}
    discriminator(R, out)
    generator(R, out)
    np.savez_compressed(os.path.join(gu.GOLDEN_DIR, "highres.npz"), **{k: np.asarray(v) for k, v in out.items()})
    w = max(len(n) for n, _ in report)
    with open(os.path.join(gu.GOLDEN_DIR, "HIGHRES_ORACLE_VS_REFERENCE.txt"), "w") as f:
        f.write("# oracle/stylegan2_oracle.py vs unmodified reference modules at 512^2 (norm-wise rel err), written by "
                "tools/make_highres_golden.py\n")
        f.write(f"# reference float32 vs float64: D[512] scores {out['d512_scores_ref32_err']:.3e}, "
                f"R1 {out['d512_r1_ref32_err']:.3e}\n")
        for n, e in report:
            f.write(f"{n:<{w}}  {e:.3e}\n")
    print("written", os.path.join(gu.GOLDEN_DIR, "highres.npz"))
