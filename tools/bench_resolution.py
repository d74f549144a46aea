#!/usr/bin/env python
"""Training-step throughput at 256^2, 512^2 or 1024^2 with the bench.py step recipe: CUDA graphs, R1 every 16th iteration,
with the path-length term (or without, --no-ppl).  Prints one JSON line (images/s, ms/step, batch, card, power limit, SM
clocks read in the same run).

  python tools/bench_resolution.py --resolution 512 --batch 16 [--no-ppl]
  python tools/bench_resolution.py --resolution 1024 --batch 8 --profile    # torch.profiler share per kernel family
  python tools/bench_resolution.py --probe                                  # narrow weight-gradient layers: SIMT vs tensor cores
  python tools/bench_resolution.py --resolution 1024 --max-batch 16         # largest multiple of 4 whose step fits
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

VOCAB = 1000


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return dict(zip(["name", "power_limit_w", "sm_mhz", "sm_max_mhz"], out))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_mhz": None, "sm_max_mhz": None}


def inputs(b, res, dev, seed=1234):
    g = torch.Generator().manual_seed(seed)
    batches = [(torch.rand(b, 3, res, res, generator=g).mul_(2).sub_(1).to(dev),
                torch.rand(b, 6, res, res, generator=g).mul_(2).sub_(1).to(dev),
                torch.randint(0, VOCAB, (b,), generator=g).to(dev)) for _ in range(2)]
    flm = torch.cat([torch.randn(b, 150, generator=g), (torch.rand(b, 6, generator=g) * 2 - 1) * 0.3,
                     torch.rand(b, 1, generator=g) * 3 + 7, (torch.rand(b, 2, generator=g) * 2 - 1) * 0.02], 1).to(dev)
    return batches, flm


def step_time(res, b, ppl, steps, warmup, texture, graph=True):
    """ms per iteration over `steps` iterations (one R1 iteration per 16, as bench.py)."""
    from gif_b200.train_step import GifTrainer
    dev = torch.device("cuda:0")
    tr = GifTrainer(dev, res, VOCAB, r1_every=16, ppl=ppl, seed=0, texture_loss=b if texture else False)
    batches, flm = inputs(b, res, dev)
    extra = (flm,) if texture else ()

    def run(n):
        for s in range(n):
            tr.train_iteration(*batches[s % 2], *extra)

    tr.iteration = 16 - warmup
    run(warmup)
    if graph:
        tr.capture(b, res)
        tr.iteration = 14
        run(2)
    torch.cuda.synchronize()
    tr.iteration = 16 - 1 - (steps - 1) % 16 if steps < 16 else 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run(steps)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return ms


def family(name):
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"^(gifb200::)?(\(anonymous namespace\)::)?", "", name)
    return re.split(r"[<(]", name)[0]


def profile(res, b, ppl, texture):
    """Eager iterations (one with R1) under torch.profiler: share of device time per kernel family and SIMT launches."""
    from torch.profiler import ProfilerActivity, profile as tprofile

    from gif_b200.train_step import GifTrainer
    dev = torch.device("cuda:0")
    tr = GifTrainer(dev, res, VOCAB, r1_every=2, ppl=ppl, seed=0, texture_loss=b if texture else False)
    batches, flm = inputs(b, res, dev)
    extra = (flm,) if texture else ()
    tr.train_iteration(*batches[0], *extra)
    torch.cuda.synchronize()
    from gif_b200 import ops
    from gif_b200._lib import lib
    ops.PROFILE = []            # eager launches record their shapes
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(2):
            tr.train_iteration(*batches[s % 2], *extra)
        torch.cuda.synchronize()
    shapes, ops.PROFILE = ops.PROFILE, None
    simt_wgrad = set()
    for *_, cfg in shapes:
        kind, mode, B, Hi, Wi, Ci, Co, k = cfg
        Ho, Wo = ops.conv_out_size(Hi, k, mode), ops.conv_out_size(Wi, k, mode)
        if kind == "wgrad" and lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, 0) == 1:
            simt_wgrad.add(str(cfg[1:]))
    fam, simt = collections.Counter(), collections.Counter()
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        t = e.device_time if hasattr(e, "device_time") else e.cuda_time
        fam[family(e.name)] += t
        if "simt_kernel" in e.name:
            simt[family(e.name)] += 1
    total = sum(fam.values())
    return {"device_ms_per_2_iterations": round(total / 1e3, 2),
            "share": {k: round(v / total, 4) for k, v in fam.most_common(20)},
            "simt_launches": dict(simt), "simt_wgrad_shapes_mode_B_Hi_Wi_Ci_Co_k": sorted(simt_wgrad)}


# (name, B, Hi, Wi, Ci, Ho, Wo, Co, k, mode): the weight gradients whose small side has 32 or 64 channels
PROBE = [
    ("G512 progression.7.st_cv2 64->64 / D conv1 64->64", 16, 512, 512, 64, 512, 512, 64, 3, 0),
    ("G512 noise conv 32->64", 16, 512, 512, 32, 512, 512, 64, 3, 0),
    ("G1024 progression.8.st_cv1 64->32 (T2)", 8, 512, 512, 64, 1025, 1025, 32, 3, 2),
    ("D512 stem 32->64 1x1", 16, 512, 512, 32, 512, 512, 64, 1, 0),
    ("D1024 stem 32->32 1x1", 8, 1024, 1024, 32, 1024, 1024, 32, 1, 0),
    ("D1024 ResBlock(32->64).conv2 (S2)", 8, 1025, 1025, 32, 512, 512, 64, 3, 1),
    ("D1024 ResBlock(32->64).skip 1x1", 8, 512, 512, 32, 512, 512, 64, 1, 0),
]


def probe(reps=10):
    from gif_b200 import ops
    dev = torch.device("cuda:0")
    rows = []
    for name, B, Hi, Wi, Ci, Ho, Wo, Co, k, mode in PROBE:
        x = ops._round_tf32_raw(torch.randn(B, Hi, Wi, Ci, device=dev))
        gy = ops._round_tf32_raw(torch.randn(B, Ho, Wo, Co, device=dev))
        row = {"layer": name, "batch": B}
        for impl in (1, 2, 3):
            old = (ops.CONV_IMPL, ops.WGRAD_IMPL)
            ops.CONV_IMPL, ops.WGRAD_IMPL = {1: (1, 1), 2: (0, 2), 3: (3, 3)}[impl]
            try:
                for _ in range(2):
                    ops._wgrad_raw(x, gy, k, mode, False, False)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    ops._wgrad_raw(x, gy, k, mode, False, False)
                e1.record()
                torch.cuda.synchronize()
            finally:
                ops.CONV_IMPL, ops.WGRAD_IMPL = old
            ms = e0.elapsed_time(e1) / reps
            sites = B * (Hi * Wi if mode == 2 else Ho * Wo)
            row[f"impl{impl}_ms"] = round(ms, 3)
            row[f"impl{impl}_tflops"] = round(2.0 * sites * Ci * Co * k * k / ms / 1e9, 1)
        rows.append(row)
        del x, gy
    return rows


def fits(res, b, precision):
    """True when a captured step at this batch runs (its own process, so that an out-of-memory leaves nothing behind)."""
    cmd = [sys.executable, os.path.abspath(__file__), "--resolution", str(res), "--batch", str(b), "--steps", "2",
           "--warmup", "2", "--precision", precision]
    try:
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    except subprocess.TimeoutExpired:
        return False
    return r.returncode == 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolution", type=int, default=512, choices=[256, 512, 1024])
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="bf16x3", choices=["tf32", "bf16x3"])
    ap.add_argument("--texture-loss", action="store_true")
    ap.add_argument("--no-ppl", action="store_true", help="drop the path-length term from the G step")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--probe", action="store_true")
    ap.add_argument("--max-batch", type=int, default=0, metavar="N", help="largest multiple of 4 up to N whose step fits")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_resolution.py needs a GPU"
    assert args.batch % 4 == 0, "minibatch standard deviation groups 4 images: the per-GPU batch is a multiple of 4"
    from gif_b200 import ops
    ops.set_precision(args.precision)
    out = {"resolution": args.resolution, "batch": args.batch, "precision": args.precision, "texture_loss": args.texture_loss,
           "path_length_reg": not args.no_ppl}
    if args.probe:
        out = {"probe": probe(), "precision": "impl 1 = exact fp32 SIMT, 2 = tf32, 3 = bf16x3"}
    elif args.max_batch:
        ok = [b for b in range(4, args.max_batch + 1, 4) if fits(args.resolution, b, args.precision)]
        out["max_batch"] = max(ok) if ok else None
        out["fits"] = ok
        del out["batch"]
    elif args.profile:
        out["profile"] = profile(args.resolution, args.batch, not args.no_ppl, args.texture_loss)
    else:
        ms = step_time(args.resolution, args.batch, not args.no_ppl, args.steps, args.warmup, args.texture_loss)
        out.update(ms_per_step=round(ms, 2), images_per_s=round(args.batch * 1000.0 / ms, 2))
        out["peak_mem_gb"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)
    out["card"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
