"""Measures the real images' FID statistics pass (gif_b200/fid_real.py) on a seeded folder of --n photo-like 1024^2 PNGs at
resolution --resolution (256 by default), with the card's name, power limit and SM clock read in the same run:

  * host CPU seconds per batch of 32 for read + parse + inflate (one thread, ``time.process_time``);
  * device ms per batch for the pinned upload + unfilter + bicubic resize (``fid_real.device_batch``), and for the
    Inception features of the uint8 batch, each timed with CUDA events over the folder's batches;
  * end-to-end images/s of ``real_image_statistics`` against the reference's procedure in the same run (Pillow open +
    resize on the host, float32 / 255, upload, then the same network), alternating, --repeats times each.  The two give
    bitwise the same statistics (the uint8 input resize is bitwise the float one), which is checked.

    python tools/bench_fid_real.py [--n 160] [--resolution 256] [--out result.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from tools.bench_resolution import card  # noqa: E402


def write_folder(d, n, size, seed=7000):
    from gif_b200.synth_images import photo

    def one(i):
        p = os.path.join(d, f"{i:05d}.png")
        photo(size, size, seed + i).save(p)
        return p
    with ThreadPoolExecutor(os.cpu_count() or 4) as pool:
        return list(pool.map(one, range(n)))


def reference_procedure(files, R, net, dims, bs, dev):
    """fid_score.get_activations' loop (fid_score.py:100-118) feeding the same network, statistics reduced on the device."""
    from gif_b200.fid import ActivationStatistics, compute_activation_batch
    stats = ActivationStatistics(dims, dev)
    with torch.no_grad():
        for i in range(0, len(files) // bs * bs, bs):
            imgs = []
            for f in files[i:i + bs]:
                img = Image.open(f)
                if R != 299:
                    img = img.resize((R, R))
                imgs.append(np.array(img).astype(np.float32))
            a = np.array(imgs).transpose((0, 3, 1, 2))
            a /= 255
            stats.update(compute_activation_batch(net, torch.from_numpy(a).to(dev)))
    return stats.finalize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=160, help="PNGs in the folder (whole batches of 32 are used)")
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--resolution", type=int, default=256)
    ap.add_argument("--dims", type=int, default=2048)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fid_real measures the device pass: it needs a CUDA device")
    from gif_b200 import fid_real, ops
    from gif_b200.fid import compute_activation_batch
    from gif_b200.inception import InceptionV3
    from oracle import inception_oracle as IO
    dev = torch.device("cuda:0")
    net = InceptionV3([InceptionV3.BLOCK_INDEX_BY_DIM[a.dims]], weights=IO.seeded_state_dict(2015)).to(dev)
    bs, R = fid_real.BATCH_SIZE, a.resolution
    res = {"card": card(), "precision": ops.get_precision(), "n_images": a.n // bs * bs, "size": a.size, "resolution": R,
           "batch": bs, "host_threads": min(32, os.cpu_count() or 1)}
    with tempfile.TemporaryDirectory() as d:
        write_folder(d, a.n, a.size)
        files = fid_real.real_image_files(d)
        res["png_mb_per_image"] = sum(os.path.getsize(f) for f in files) / len(files) / 1e6
        batches = [files[i:i + bs] for i in range(0, len(files), bs)]

        cpu = []
        loaded = []
        for b in batches:                                           # host side, one thread
            t0 = time.process_time()
            loaded.append([fid_real.load_png(f) for f in b])
            cpu.append(time.process_time() - t0)
        res["host_cpu_s_per_batch_parse_inflate"] = float(np.mean(cpu))

        status = torch.zeros(bs, dtype=torch.int32, device=dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        dec_ms, inc_ms = [], []
        with torch.no_grad():
            for rep in range(2):                                    # the first pass warms up every shape
                for b, ld in zip(batches, loaded):
                    torch.cuda.synchronize()
                    ev[0].record()
                    x = fid_real.device_batch(b, ld, R, status, dev)
                    ev[1].record()
                    compute_activation_batch(net, x)
                    ev[2].record()
                    torch.cuda.synchronize()
                    if rep:
                        dec_ms.append(ev[0].elapsed_time(ev[1]))
                        inc_ms.append(ev[1].elapsed_time(ev[2]))
        res["device_ms_per_batch_upload_unfilter_resize"] = float(np.mean(dec_ms))
        res["device_ms_per_batch_inception"] = float(np.mean(inc_ms))
        del loaded

        ours, ref = [], []
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m1, s1 = fid_real.real_image_statistics(d, R, net, a.dims)
            torch.cuda.synchronize()
            ours.append(len(files) / (time.perf_counter() - t0))
            t0 = time.perf_counter()
            m2, s2 = reference_procedure(files, R, net, a.dims, bs, dev)
            torch.cuda.synchronize()
            ref.append(len(files) / (time.perf_counter() - t0))
        res["images_per_s_device_pipeline"] = ours
        res["images_per_s_reference_procedure"] = ref
        res["statistics_bitwise_equal"] = bool(torch.equal(m1, m2) and torch.equal(s1, s2))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
