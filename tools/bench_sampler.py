#!/usr/bin/env python
"""Rows-to-bytes sampling throughput (images/s) at 256^2: DECA rows on the device in, uint8 images out, for three arms
alternated round by round in one run:
    graphs   FlameSampler(graphs=True): one CUDA-graph replay per batch
    eager    FlameSampler(graphs=False): the same kernels launched from Python
    compose  what the project offered before FlameSampler: eye_centering.position_to_given_location,
             DecaConditionRenderer (condition in [-1, 1]) -> host -> inference.get_images_from_flame_params -> numpy bytes
             (it renders no mesh picture, which the other two arms do)
for batch 32 and 16 in bf16x3 and tf32, seeded weights, synthetic FLAME.  Prints one JSON line per configuration and the
card's name, power limit and SM clock read in the same run.

  python tools/bench_sampler.py [--n 256] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256, help="rows per timed window")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    from sample_faces import draw_identities, draw_rows
    from gif_b200 import ops
    from gif_b200.conditions import DecaConditionRenderer
    from gif_b200.eye_centering import position_to_given_location
    from gif_b200.flame import FLAME, FLAMETex
    from gif_b200.flame_synth import flame_uv, synthetic_flame_model, synthetic_texture_space
    from gif_b200.inference import get_images_from_flame_params
    from gif_b200.model.stg2_generator import StyledGenerator
    from gif_b200.sampler import FlameSampler
    dev = torch.device("cuda:0")
    flame = FLAME.from_arrays(synthetic_flame_model()).to(dev)
    mean, basis = synthetic_texture_space(512, 50)
    cr = DecaConditionRenderer(flame, FLAMETex(mean=mean, basis=basis).to(dev), *flame_uv())
    torch.manual_seed(0)
    G = StyledGenerator(embedding_vocab_size=VOCAB, rendered_flame_ascondition=True, normal_maps_as_cond=True).to(dev).eval()
    rows = torch.from_numpy(draw_rows(args.n, 0)).to(dev)
    ids = torch.from_numpy(draw_identities(args.n, VOCAB, 0)).to(dev)
    print(json.dumps({"card": card()}), flush=True)
    for precision in ("bf16x3", "tf32"):
        ops.set_precision(precision)
        for batch in (32, 16):
            graphs = FlameSampler(G, cr, 256, batch, graphs=True)
            eager = FlameSampler(G, cr, 256, batch, graphs=False)

            def compose():
                centred = position_to_given_location(flame, rows.clone())
                cond = cr(centred).cpu()
                img = get_images_from_flame_params(cond, None, G, 6, 1, ids.cpu(), batch_size=batch, device=dev)
                return (np.clip((img.numpy() + 1) / 2, 0, 1) * 255).astype(np.uint8)

            arms = {"graphs": lambda: graphs.sample(rows, ids)["images"], "eager": lambda: eager.sample(rows, ids)["images"],
                    "compose": compose}
            for fn in arms.values():                                 # warm-up (and the graphs' capture)
                fn()
            torch.cuda.synchronize()
            times = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    times[k].append(time.perf_counter() - t0)
            res = {k: round(args.n / statistics.median(v), 1) for k, v in times.items()}
            spread = {k: round((max(v) - min(v)) / statistics.median(v), 3) for k, v in times.items()}
            print(json.dumps({"precision": precision, "batch": batch, "resolution": 256, "rows": args.n,
                              "images_per_s": res, "rel_spread": spread, "rounds": args.rounds}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
