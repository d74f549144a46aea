"""Multiscale image LMDB throughput: images/s of ``prepare_multiscale_lmdb`` over a seeded folder of 1024^2 PNGs
(``synth_images.png_folder``), against the reference's recipe (Pillow decode, torchvision resize(LANCZOS) + center_crop and
Pillow's JPEG q100 for each size, one image per task) on a process pool of the host's cores, in the same run.

The device path is also taken apart: host read + parse + inflate of every file on the thread pool (wall), the device work
per batch (decode, the eight resizes and encodes, the byte counts and bytes copied back; host clock around work that ends
in a synchronise), and the LMDB writes.  Prints the card's name and power limit, read in the same run; prints one JSON line
and, with --out, also writes it to that file."""
import argparse
import io
import json
import multiprocessing
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def reference_worker(args):
    path, sizes = args
    from PIL import Image
    from torchvision.transforms import functional as tv
    img = Image.open(path).convert("RGB")
    out = []
    for s in sizes:
        b = io.BytesIO()
        tv.center_crop(tv.resize(img, s, Image.LANCZOS), s).save(b, format="jpeg", quality=100)
        out.append(b.getvalue())
    return out


def profile_batch(P, encode_jpeg_batch, loaded):
    """Device time (ms) per kernel / copy name over one batch: decode, then the resizes and encodes of every size."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda")
    for _ in range(2):                                   # the first pass warms up
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            groups = P.decoded_groups(loaded, dev)
            for s in P.SIZES:
                encode_jpeg_batch(P.resized_crops(groups, len(loaded), s))
            torch.cuda.synchronize()
    rows = [(e.key, e.device_time_total / 1e3, e.count) for e in prof.key_averages() if e.device_time_total > 0]
    return {k: {"ms": round(t, 3), "calls": c} for k, t, c in sorted(rows, key=lambda r: -r[1])[:25]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256, help="images in the seeded folder")
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--threads", type=int, default=None)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--profile", action="store_true",
                    help="afterwards, one batch under torch.profiler: device time per kernel (a run of its own)")
    a = ap.parse_args()
    import torch
    from gif_b200 import prepare_images as P
    from gif_b200.data import LmdbWriter, image_key
    from gif_b200.image_encode import encode_jpeg_batch
    from gif_b200.synth_images import png_folder
    if not torch.cuda.is_available():
        raise SystemExit("bench_prepare measures the device path: it needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card, "n": a.n, "size": a.size, "batch_size": a.batch_size, "sizes": list(P.SIZES),
           "host_cpus": os.cpu_count()}
    with tempfile.TemporaryDirectory() as tmp:
        png_folder(os.path.join(tmp, "src", "images"), a.n, a.size, seed=0)
        files = P.image_files(os.path.join(tmp, "src"))
        threads = a.threads or min(32, os.cpu_count() or 1)

        # warm-up: module load, coefficient tables, kernels
        P.prepare_multiscale_lmdb(os.path.join(tmp, "src"), os.path.join(tmp, "warm"), batch_size=a.batch_size,
                                  threads=threads)
        t0 = time.perf_counter()
        P.prepare_multiscale_lmdb(os.path.join(tmp, "src"), os.path.join(tmp, "db"), batch_size=a.batch_size, threads=threads)
        res["device_path_s"] = time.perf_counter() - t0
        res["device_path_images_per_s"] = a.n / res["device_path_s"]

        # the stages on their own
        with ThreadPoolExecutor(threads) as pool:
            t0 = time.perf_counter()
            loaded = list(pool.map(P.load_image, files))
            res["host_read_inflate_s"] = time.perf_counter() - t0
        values = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(0, len(files), a.batch_size):
            names = files[k:k + a.batch_size]
            groups = P.decoded_groups(loaded[k:k + a.batch_size], torch.device("cuda"))
            for s in P.SIZES:
                blobs = encode_jpeg_batch(P.resized_crops(groups, len(names), s))
                values += [(image_key(s, k + i), b) for i, b in enumerate(blobs)]
        torch.cuda.synchronize()
        res["device_s"] = time.perf_counter() - t0
        res["device_images_per_s"] = a.n / res["device_s"]
        res["bytes_per_image"] = sum(len(v) for _, v in values) / a.n
        t0 = time.perf_counter()
        with LmdbWriter(os.path.join(tmp, "db2")) as w:
            for k, v in values:
                w.put(k, v)
        res["lmdb_write_s"] = time.perf_counter() - t0

        # the reference's recipe on a process pool of the host's cores
        with multiprocessing.get_context("spawn").Pool(os.cpu_count()) as pool:
            pool.map(reference_worker, [(files[0], P.SIZES)] * (os.cpu_count() or 1))      # warm the workers
            t0 = time.perf_counter()
            ref = pool.map(reference_worker, [(f, P.SIZES) for f in files], chunksize=1)
            res["reference_s"] = time.perf_counter() - t0
        res["reference_images_per_s"] = a.n / res["reference_s"]
        mine = dict(values)
        res["equal_to_reference"] = all(mine[image_key(s, i)] == ref[i][j] for i in range(a.n) for j, s in enumerate(P.SIZES))
        if a.profile:
            res["profile_ms_per_batch"] = profile_batch(P, encode_jpeg_batch, loaded[:a.batch_size])
    res["card_after"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                                       capture_output=True, text=True).stdout.strip()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
