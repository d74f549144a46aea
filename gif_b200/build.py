"""Builds gif_b200/libgifb200.so (hand-written CUDA for sm_90a + the C ABI of include/gifb200.h) with nvcc.

In-tree build: the .so lands next to this file, so the package is importable from the source tree.
``python -m gif_b200.build`` or ``__graft_entry__.build()``.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libgifb200.so")
SOURCES = ["elementwise.cu", "optim.cu", "upfirdn2d.cu", "sgemm.cu", "conv_simt.cu", "conv_tc.cu", "conv_wgrad_tc.cu", "conv_api.cu", "conv_ex.cu", "pool_resize.cu", "rasterize.cu", "render.cu", "flame.cu", "texture.cu", "image_decode.cu", "jpeg_encode.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
         "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]


def _stamp(path):
    h = hashlib.sha1()
    for f in [path, os.path.join(ROOT, "include", "gifb200.h")] + \
            [os.path.join(CSRC, x) for x in sorted(os.listdir(CSRC)) if x.endswith(".cuh")]:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _current():
    """True when the library and every object exist and match the sources and flags (nothing to do, nothing written)."""
    if not os.path.isfile(LIB):
        return False
    for src in SOURCES:
        stamp_file = os.path.join(OBJ, src.replace(".cu", ".o")) + ".stamp"
        if not os.path.isfile(stamp_file) or open(stamp_file).read() != _stamp(os.path.join(CSRC, src)):
            return False
    return True


def build(verbose=False, force=False):
    """Incremental (content-hash stamps).  Safe under ``torchrun``: an exclusive file lock serialises concurrent builders
    (all ranks import the package at once), and every object / the library is written to a temporary name and renamed into
    place, so a process that is not building never sees a half-written file.  A current build is left untouched without
    taking the lock, so an already built tree may be read-only."""
    import fcntl
    if not force and _current():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    with open(os.path.join(OBJ, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(verbose, force)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose, force):
    objs, rebuilt = [], False
    for src in SOURCES:
        path = os.path.join(CSRC, src)
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        stamp_file = obj + ".stamp"
        stamp = _stamp(path)
        if force or not os.path.isfile(obj) or not os.path.isfile(stamp_file) or open(stamp_file).read() != stamp:
            tmp = obj + f".tmp{os.getpid()}"
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", path, "-o", tmp]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                raise RuntimeError(f"nvcc failed on {src}")
            if verbose:
                print(r.stderr)
            os.replace(tmp, obj)
            with open(stamp_file + ".tmp", "w") as f:
                f.write(stamp)
            os.replace(stamp_file + ".tmp", stamp_file)
            rebuilt = True
        objs.append(obj)
    if rebuilt or not os.path.isfile(LIB):
        tmp = LIB + f".tmp{os.getpid()}"
        cmd = [NVCC, "-shared", "-o", tmp] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
