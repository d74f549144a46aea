"""Build the multiscale training-image LMDB from an image folder (``ImageFolder`` layout: class directories of PNG / JPEG
files), on the device: the LMDB the reference's prepare_lmdb/prepare_ffhq_multiscale_dataset.py writes, byte for byte.

    python tools/prepare_ffhq_lmdb.py DATASET_PATH --out DIR [--sizes 8 16 ... 1024] [--batch-size 32] [--threads N]"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main(argv=None):
    from gif_b200.prepare_images import SIZES, prepare_multiscale_lmdb
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("path", help="image folder: class directories of PNG / baseline JPEG files")
    ap.add_argument("--out", required=True, help="LMDB directory to create (must not exist)")
    ap.add_argument("--sizes", type=int, nargs="+", default=list(SIZES))
    ap.add_argument("--quality", type=int, default=100)
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--threads", type=int, default=None, help="host threads reading and inflating (default: CPU count, <= 32)")
    a = ap.parse_args(argv)
    t0 = time.perf_counter()
    n = prepare_multiscale_lmdb(a.path, a.out, sizes=tuple(a.sizes), quality=a.quality, batch_size=a.batch_size,
                                threads=a.threads)
    print(f"{n} images at sizes {a.sizes} -> {a.out} in {time.perf_counter() - t0:.1f} s")


if __name__ == "__main__":
    main()
