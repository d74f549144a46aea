"""Input-pipeline measurement.

1. Host CPU seconds per batch: ``GifLmdbDataset`` items (PIL decode, the work of PinnedBatchLoader's thread) and
   DeviceBatchLoader's host side (LMDB read, parsing, PNG inflate on its pool).  ``time.process_time`` sums every thread
   of the process; torch runs with one intra-op thread so that OpenMP workers spin-waiting inside the PIL path's small
   float ops are not counted as decode work.
2. Device decode time per batch (CUDA events), split into JPEG (for several entropy chunk sizes), PNG and resize, with
   the bytes each pass reads.
3. ``--trainer``: GifTrainer images/s at 256^2 batch 32 (bf16x3, CUDA graphs, no path-length term) fed by DeviceBatchLoader
   against the same step fed from pinned host tensors, alternating, three runs of each.
4. ``--conditions render``: the same legs with the conditions rendered on the device from DECA rows
   (DeviceBatchLoader(conditions=DecaConditionRenderer), synthetic FLAME model, analytic 512^2 x 50 texture space) next to
   the PNG path: host CPU s/batch, device ms/batch of the render against the PNG unfilter, and a third trainer arm.

The synthetic LMDBs follow the reference's writers (JPEG q100 4:2:0 real images, PNG renders at 256^2).  Prints the card,
its power limit and clocks read in the same run; writes JSON to --out."""
import argparse
import itertools
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def cpu_per_batch(fn, reps):
    fn()
    t0 = time.process_time()
    for _ in range(reps):
        fn()
    return (time.process_time() - t0) / reps


def event_ms(fn, iters=20):
    for _ in range(3):
        fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def condition_renderer(rr):
    from gif_b200.conditions import DecaConditionRenderer
    from gif_b200.flame import FLAME, FLAMETex
    from gif_b200.flame_synth import flame_uv, synthetic_flame_model, synthetic_texture_space
    mean, basis = synthetic_texture_space(512, 50)
    return DecaConditionRenderer(FLAME.from_arrays(synthetic_flame_model()).cuda(), FLAMETex(mean=mean, basis=basis).cuda(),
                                 *flame_uv(), image_size=rr)


def render_leg(row, real, R, bs, reps, cr):
    """Host CPU s/batch of the render-fed loader and device ms/batch of the render (FLAME, FLAMETex, rasteriser, shading)."""
    from concurrent.futures import ThreadPoolExecutor
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset
    from gif_b200.flame_synth import synthetic_deca_params
    params = synthetic_deca_params(bs, 3).numpy()
    ds = GifLmdbDataset(real, None, params, resolution=R, rend_flm_res=256)
    loader = DeviceBatchLoader(ds, bs, conditions=cr)
    ids = list(range(bs))
    with ThreadPoolExecutor(loader.threads) as pool:
        row["render_loader_host_cpu_s"] = cpu_per_batch(lambda: loader.host_batch(ids, pool), reps)
    raw = torch.from_numpy(params).cuda()
    out = torch.empty(2 * bs, 256, 256, 3, dtype=torch.uint8, device="cuda")
    row["render_ms"] = event_ms(lambda: cr.render_u8(raw, out=out))
    row["flametex_ms"] = event_ms(lambda: cr.flametex(raw[:, 159:209]))
    row["flametex_bytes"] = 256 * 256 * 3 * 51 * 4 + bs * 3 * 256 * 256 * 4


def decode_leg(R, bs, reps, chunks, cr=None):
    from concurrent.futures import ThreadPoolExecutor
    from gif_b200 import image_decode as I
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset, image_key, normal_map_key
    from gif_b200.synth_images import build_lmdbs
    with tempfile.TemporaryDirectory() as tmp:
        real, rend = build_lmdbs(tmp, bs, R, 256)
        ds = GifLmdbDataset(real, rend, np.zeros((bs, 8), np.float32), resolution=R, rend_flm_res=256)
        ids = list(range(bs))
        pil = cpu_per_batch(lambda: [ds[i] for i in ids], reps)
        loader = DeviceBatchLoader(ds, bs)
        with ThreadPoolExecutor(loader.threads) as pool:
            dev_host = cpu_per_batch(lambda: loader.host_batch(ids, pool), reps)
        row = {"resolution": R, "batch": bs, "pil_cpu_s": pil, "device_loader_host_cpu_s": dev_host,
               "host_cpu_ratio": pil / dev_host}
        if not torch.cuda.is_available():
            return row
        # each kernel on its own: the loader's records, packed and uploaded here
        jpegs = [I.host_decode(ds.real.get(image_key(R, i)), str(i)) for i in ids]
        pngs = [I.host_decode(ds.rend.get(key(256, i)), str(i)) for key in (image_key, normal_map_key) for i in ids]
        to_dev = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).cuda()
        jb = I.JpegBatch([im.data for im in jpegs])
        data = to_dev(jb.data)
        out = torch.empty(jb.out_bytes, dtype=torch.uint8, device="cuda")
        st = torch.zeros(3 * bs, dtype=torch.int32, device="cuda")
        ref = None
        for cb in chunks:
            b = I.JpegBatch([im.data for im in jpegs], cb)
            ints = torch.from_numpy(b.ints).cuda()
            ws = torch.empty(b.workspace_bytes, dtype=torch.uint8, device="cuda")
            row[f"jpeg_ms_chunk{cb}"] = event_ms(lambda: b.launch(data, ints, out, st[:bs], ws))
            ref = out.clone() if ref is None else ref
            assert torch.equal(out, ref) and (st.cpu() == 0).all(), cb     # every chunk size decodes the same bits
        pb = I.PngBatch([(im.w, im.h, im.bpp, b"") for im in pngs], [im.data for im in pngs])
        scan, desc = to_dev(b"".join(im.data for im in pngs)), torch.from_numpy(pb.desc).cuda()
        rend_u8 = torch.empty(2 * bs, 256, 256, 3, dtype=torch.uint8, device="cuda")
        work = scan.clone()
        row["png_ms"] = event_ms(lambda: (work.copy_(scan), pb.launch(work, desc, rend_u8, st[bs:])))
        if R != 256:
            row["resize_ms"] = event_ms(lambda: I.resize_bicubic_u8(rend_u8, R))
        row["jpeg_entropy_bytes"], row["png_inflated_bytes"] = len(jb.data), pb.data_bytes
        if cr is not None:
            render_leg(row, real, R, bs, reps, cr)
        return row


def trainer_leg(runs, steps, R=256, B=32, vocab=1000, cr=None):
    from gif_b200 import ops
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset
    from gif_b200.synth_images import build_lmdbs
    from gif_b200.train_step import GifTrainer
    dev = torch.device("cuda")
    ops.set_precision("bf16x3")
    trainer = GifTrainer(dev, R, vocab, r1_every=16, ppl=False, seed=0)
    gen = torch.Generator().manual_seed(1234)
    host = [(torch.rand(B, 3, R, R, generator=gen).mul_(2).sub_(1).pin_memory(),
             torch.rand(B, 6, R, R, generator=gen).mul_(2).sub_(1).pin_memory(),
             torch.randint(0, vocab, (B,), generator=gen).pin_memory()) for _ in range(4)]
    trainer.iteration = 16 - 3
    for s in range(3):
        trainer.train_iteration(*(t.to(dev) for t in host[s]))
    torch.cuda.synchronize()
    trainer.capture(B, R)
    trainer.iteration = 14
    for s in range(2):
        trainer.train_iteration(*host[s])
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        real, rend = build_lmdbs(tmp, 4 * B, R, 256)
        ds = GifLmdbDataset(real, rend, np.zeros((4 * B, 8), np.float32), resolution=R, rend_flm_res=256)
        loader = DeviceBatchLoader(ds, B)
        batches = itertools.chain.from_iterable(iter(loader) for _ in itertools.count())
        first = next(batches)
        arms = {"pinned": None, "device_loader": [batches, first]}
        if cr is not None:
            from gif_b200.flame_synth import synthetic_deca_params
            rds = GifLmdbDataset(real, None, synthetic_deca_params(4 * B, 5).numpy(), resolution=R, rend_flm_res=256)
            rloader = DeviceBatchLoader(rds, B, conditions=cr)
            rb = itertools.chain.from_iterable(iter(rloader) for _ in itertools.count())
            arms["render_loader"] = [rb, next(rb)]

        def pinned():
            for s in range(steps):
                trainer.train_iteration(*host[s % 4])

        def fed(arm):
            def run():
                src, first = arm
                for s in range(steps):
                    real_b, cond_b, _, idx_b = first if s == 0 else next(src)
                    trainer.train_iteration(real_b, cond_b, idx_b)
                arm[1] = next(src)
            return run

        fns = [(name, pinned if arm is None else fed(arm)) for name, arm in arms.items()]
        res = {name: [] for name in arms}
        for _ in range(runs):
            for name, fn in fns:
                trainer.iteration = 0                  # one R1 iteration in every window of 16
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                res[name].append(B * steps / (time.perf_counter() - t0))
        return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="256:32,512:16,1024:8")
    ap.add_argument("--chunks", default="512,1024,2048,4096")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--trainer", action="store_true")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--conditions", choices=("lmdb", "render"), default="lmdb",
                    help="render: also measure conditions rendered on the device from DECA rows")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.set_num_threads(1)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip() if torch.cuda.is_available() else "no GPU"
    res = {"card": card, "configs": []}
    cr = condition_renderer(256) if args.conditions == "render" else None
    for cfg in args.configs.split(","):
        R, bs = map(int, cfg.split(":"))
        row = decode_leg(R, bs, args.reps, [int(c) for c in args.chunks.split(",")], cr)
        res["configs"].append(row)
        print(json.dumps(row), flush=True)
    if args.trainer:
        res["trainer_images_per_s"] = trainer_leg(args.runs, args.steps, cr=cr)
        print(json.dumps(res["trainer_images_per_s"]), flush=True)
    res["card_after"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                                       capture_output=True, text=True).stdout.strip() if torch.cuda.is_available() else ""
    print("card:", card, "| after:", res["card_after"])
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
