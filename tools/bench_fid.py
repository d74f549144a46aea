#!/usr/bin/env python
"""FID feature extraction on the library's own kernels (gif_b200.inception.InceptionV3).  Prints one JSON line with the card,
its power limit and clocks read in the same run, and:

  * images/s of feature extraction (block 3, 2048-d) from 256^2 inputs at batch 32 and 128, in fp32, tf32 and bf16x3;
  * the same seeded weights through torch / cuDNN (the float32 functional oracle) in fp32 and tf32, as a baseline only;
  * per layer family (1x1, 3x3, 5x5, 1x7/7x1, 1x3/3x1): kernel time of gifb200_conv2d_ex at batch 32 and the achieved
    TFLOP/s (the multiply-adds per image are computed from the layer shapes below: about 5.71 G);
  * wall time of FidComputer.get_fid on --fid-images seeded 256^2 generator images (generator + features + statistics).

  python tools/bench_fid.py [--fid-images 10000] [--profile]
"""
import argparse
import collections
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

from tools.bench_resolution import card  # noqa: E402


def layer_shapes(hw=299):
    """(name, Ci, Co, kh, kw, stride, pad_h, pad_w, Hi, Wi, Ho, Wo) of every convolution for a hw x hw input."""
    from gif_b200.inception import BLOCKS
    out = []
    for mods in BLOCKS:
        for _, convs in mods:
            for name, ci, co, kh, kw, s, ph, pw in convs:
                Hi = _input_size(name, hw)
                Ho = (Hi + 2 * ph - kh) // s + 1
                Wo = (Hi + 2 * pw - kw) // s + 1
                out.append((name, ci, co, kh, kw, s, ph, pw, Hi, Hi, Ho, Wo))
    return out


def _input_size(name, hw):
    c1 = (hw - 3) // 2 + 1
    c2 = c1 - 2
    p1 = (c2 - 3) // 2 + 1
    c4 = p1 - 2
    p2 = (c4 - 3) // 2 + 1
    m6 = (p2 - 3) // 2 + 1
    m7 = (m6 - 3) // 2 + 1
    table = [("Conv2d_1a", hw), ("Conv2d_2a", c1), ("Conv2d_2b", c2), ("Conv2d_3b", p1), ("Conv2d_4a", p1),
             ("Mixed_5", p2), ("Mixed_6a", p2), ("Mixed_6", m6), ("Mixed_7a", m6), ("Mixed_7", m7)]
    return next(v for k, v in table if name.startswith(k))


def family(kh, kw):
    return {(1, 1): "1x1", (3, 3): "3x3", (5, 5): "5x5", (1, 7): "1x7/7x1", (7, 1): "1x7/7x1", (1, 3): "1x3/3x1",
            (3, 1): "1x3/3x1"}[(kh, kw)]


def macs_per_image():
    return sum(ci * co * kh * kw * Ho * Wo for _, ci, co, kh, kw, _, _, _, _, _, Ho, Wo in layer_shapes())


def timed(fn, n, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fid-images", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--profile", action="store_true", help="torch.profiler kernel-time share per kernel at batch 32")
    ap.add_argument("--out", default=None, help="also write the JSON to this file")
    a = ap.parse_args()
    from gif_b200 import ops
    from gif_b200.inception import InceptionV3
    from oracle import inception_oracle as IO
    dev = torch.device("cuda:0")
    res = {"card": card(), "gmac_per_image": macs_per_image() / 1e9}
    sd = IO.seeded_state_dict(2015)
    net = InceptionV3([3], weights=sd).to(dev)
    g = torch.Generator().manual_seed(0)
    imgs = {b: torch.rand(b, 3, 256, 256, generator=g).to(dev) for b in (32, 128)}
    res["features_images_per_s"] = {}
    with torch.no_grad():
        for prec in ("fp32", "tf32", "bf16x3"):
            ops.set_precision(prec)
            for b, x in imgs.items():
                ms = timed(lambda: net(x), a.iters)
                res["features_images_per_s"][f"{prec}_b{b}"] = round(b / ms * 1e3, 1)
        ops.set_precision("tf32")
        sd32 = {k: v.float().to(dev) for k, v in sd.items()}
        res["cudnn_baseline_images_per_s"] = {}
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            for b, x in imgs.items():
                ms = timed(lambda: IO.forward(sd32, x, (3,)), a.iters)
                res["cudnn_baseline_images_per_s"][f"{'tf32' if tf32 else 'fp32'}_b{b}"] = round(b / ms * 1e3, 1)
        torch.backends.cudnn.allow_tf32 = True
        # per layer family: every convolution of a 299^2 forward at batch 32, timed alone
        fam = collections.defaultdict(lambda: collections.defaultdict(float))
        B = 32
        for prec in ("tf32", "bf16x3"):
            ops.set_precision(prec)
            for name, ci, co, kh, kw, s, ph, pw, Hi, Wi, Ho, Wo in layer_shapes():
                ci32, co32 = (ci + 31) // 32 * 32, (co + 31) // 32 * 32
                x = torch.randn(B, Hi, Wi, ci32, device=dev)
                w = torch.randn(kh * kw, co32, ci32, device=dev) * 0.05
                ws = [None, None]
                ms = timed(lambda: ops.conv2d_ex(x, w, kh, kw, s, (ph, pw), workspace=ws), 5)
                f = family(kh, kw)
                fam[prec][f + "_ms"] += ms
                fam[prec][f + "_gmac"] += B * ci * co * kh * kw * Ho * Wo / 1e9
        res["conv_families_b32"] = {p: {f: {"ms": round(d[f + "_ms"], 3), "tflops": round(2 * d[f + "_gmac"] / d[f + "_ms"], 1)}
                                        for f in sorted({k[:-3] for k in d if k.endswith("_ms")})} for p, d in fam.items()}
        if a.profile:
            ops.set_precision("bf16x3")
            x = imgs[32]
            net(x)
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                net(x)
                torch.cuda.synchronize()
            k = collections.Counter()
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    k[e.name.split("(")[0][-80:]] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            tot = sum(k.values())
            res["profile_bf16x3_b32"] = {n: round(t / tot, 4) for n, t in k.most_common(12)}
    if a.fid_images:
        res["get_fid"] = fid_wall_time(a.fid_images, dev)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


def fid_wall_time(n, dev):
    """FidComputer.get_fid on n seeded 256^2 generator images (bf16x3): generation, features and statistics, each timed."""
    import golden_util as gu
    from gif_b200 import ops
    from gif_b200.fid import FidComputer
    from gif_b200.inference import get_images_from_flame_params
    from gif_b200.model.stg2_generator import StyledGenerator
    from oracle import inception_oracle as IO
    ops.set_precision("bf16x3")
    G = StyledGenerator(embedding_vocab_size=16, rendered_flame_ascondition=True, normal_maps_as_cond=True)
    G.load_state_dict(gu.seeded_state_dict(gu.g_shapes(16), 5))
    G.to(dev)
    fc = FidComputer(dims=2048, inception_weights=IO.seeded_state_dict(2015), device=dev)
    fc.m_t, fc.s_t, fc.current_resolution = torch.zeros(2048, dtype=torch.float64), torch.eye(2048, dtype=torch.float64), 256
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    chunks = []
    with torch.no_grad():
        for i in range(0, n, 1024):                      # conditions made per chunk: 10 000 of them are 16 GB
            m = min(1024, n - i)
            cond, idx = gu.rand_uniform((m, 6, 256, 256), 1 + i), gu.randint(16, (m,), 2 + i)
            chunks.append(get_images_from_flame_params(cond, None, G, step=6, alpha=1, input_indices=idx, batch_size=32,
                                                       device=dev))
    images = torch.cat(chunks)
    del chunks
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    fid = fc.get_fid(images)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    return {"images": n, "generator_s": round(t1 - t0, 2), "features_and_fid_s": round(t2 - t1, 2),
            "total_s": round(t2 - t0, 2), "fid": fid}


if __name__ == "__main__":
    main()
