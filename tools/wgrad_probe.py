#!/usr/bin/env python
"""Single weight-gradient launches through the C ABI for timing.

    python tools/wgrad_probe.py [ns|mid|low|s2|t2] ...              tf32 kernel on the named shapes
    python tools/wgrad_probe.py --precision bf16x3 [--rounds R] [name ...]
                                                                    bf16x3 kernel on the 256^2 step's weight-gradient shapes: both
                                                                    operands from shared memory and one B tile per tap
                                                                    (GIFB200_WGRAD_X3_RS=0 GIFB200_WGRAD_HALO=0, "ss") and the
                                                                    default (S operand in registers, halo tile: "rs"), alternating
                                                                    for R rounds (one child process per path and round: the
                                                                    switches are read once)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {"ns": ("S1", 32, 256, 128, 128), "mid": ("S1", 32, 128, 256, 256), "low": ("S1", 32, 64, 512, 512),
         "s2": ("S2", 32, 257, 128, 256), "t2": ("T2", 32, 128, 256, 128)}
# (mode, batch, input resolution, Ci, Co, k): the bf16x3 weight-gradient shapes that take the most time in the 256^2
# batch-32 training step (GIFB200_SHAPE_PROFILE of bench.py), largest first
X3_CASES = {
    "s1_512_64": ("S1", 32, 64, 512, 512, 3),         # 512 -> 512 3x3 @64^2
    "s1_256_128": ("S1", 32, 128, 256, 256, 3),       # 256 -> 256 3x3 @128^2
    "s1_128_256": ("S1", 32, 256, 128, 128, 3),       # 128 -> 128 3x3 @256^2
    "s2_256_129": ("S2", 32, 129, 256, 512, 3),       # stride-2 129^2 -> 64^2
    "s2_128_257": ("S2", 32, 257, 128, 256, 3),       # stride-2 257^2 -> 128^2
    "s1_512_32": ("S1", 32, 32, 512, 512, 3),         # 512 -> 512 3x3 @32^2
    "s2_512_65": ("S2", 32, 65, 512, 512, 3),         # stride-2 65^2 -> 32^2
    "t2_512_64": ("T2", 32, 64, 512, 256, 3),         # transposed 64^2 -> 129^2
    "s1_32_256": ("S1", 32, 256, 32, 128, 3),         # 32 -> 128 3x3 @256^2 (BLOCK_N 32)
    "t2_256_128": ("T2", 32, 128, 256, 128, 3),       # transposed 128^2 -> 257^2
    "stack_32_256": ("S1", 32, 256, 32, 32, 3),       # 32 -> 32 3x3 @256^2 (STACK: the padded noise convs)
}


def _time(fn, iters=10):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _tflops(mode, b, r, ci, co, k, ms):
    from gif_b200 import ops
    ho = ops.conv_out_size(r, k, mode)
    sites = b * (r * r if mode == ops.T2 else ho * ho)
    return 2.0 * sites * ci * co * k * k / ms / 1e9


def tf32_main(names):
    import torch
    from gif_b200 import ops
    dev = torch.device("cuda:0")
    ops.set_precision("tf32")
    for n in names:
        mode, b, r, ci, co = CASES[n]
        mode = getattr(ops, mode)
        ho = ops.conv_out_size(r, 3, mode)
        x = ops._round_tf32_raw(torch.randn(b, r, r, ci, device=dev))
        gy = ops._round_tf32_raw(torch.randn(b, ho, ho, co, device=dev))
        ms = _time(lambda: ops._wgrad_raw(x, gy, 3, mode, False, False))
        print(f"{n}: {ms:.3f} ms  {_tflops(mode, b, r, ci, co, 3, ms):.1f} TFLOP/s", flush=True)


def x3_child(names):
    """One path (whatever GIFB200_WGRAD_X3_RS says): {name: ms} of the bf16x3 weight gradient on the split planes."""
    import torch
    from gif_b200 import ops
    from gif_b200._lib import lib
    dev = torch.device("cuda:0")
    ops.set_precision("bf16x3")
    out = {}
    for n in names:
        mode, b, r, ci, co, k = X3_CASES[n]
        mode = getattr(ops, mode)
        ho = ops.conv_out_size(r, k, mode)
        assert lib.gifb200_conv2d_wgrad_path(b, r, r, ci, ho, ho, co, k, mode, 3) == 3, n
        x = torch.randn(b, r, r, ci, device=dev)
        gy = torch.randn(b, ho, ho, co, device=dev)
        xp, gp = ops._planes(x), ops._planes(gy)                # split once: time the weight gradient alone
        out[n] = _time(lambda: ops._wgrad_raw(x, gy, k, mode, False, False, x_planes=xp))
        del x, gy, xp, gp
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


def x3_main(names, rounds):
    runs = {"ss": [], "rs": []}
    for _ in range(rounds):
        for path, rs in (("ss", "0"), ("rs", "1")):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--x3-child"] + names,
                               env=dict(os.environ, GIFB200_WGRAD_X3_RS=rs, GIFB200_WGRAD_HALO=rs), capture_output=True, text=True)
            if r.returncode != 0:
                sys.exit(r.stdout + r.stderr)
            runs[path].append(json.loads(r.stdout.strip().splitlines()[-1]))
    print(f"{'shape':<14} {'ss ms (min-max)':>17} {'rs ms (min-max)':>17} {'ss TFLOP/s':>11} {'rs TFLOP/s':>11} {'speed-up':>8}")
    for n in names:
        mode, b, r, ci, co, k = X3_CASES[n]
        ss, rs = [x[n] for x in runs["ss"]], [x[n] for x in runs["rs"]]
        from gif_b200 import ops
        m = getattr(ops, mode)
        print(f"{n:<14} {min(ss):7.3f}-{max(ss):7.3f}   {min(rs):7.3f}-{max(rs):7.3f}   {_tflops(m, b, r, ci, co, k, min(ss)):9.1f}  "
              f"{_tflops(m, b, r, ci, co, k, min(rs)):9.1f}  {min(ss) / min(rs):7.3f}x", flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="tf32", choices=["tf32", "bf16x3"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--x3-child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("names", nargs="*")
    a = ap.parse_args()
    if a.x3_child:
        x3_child(a.names)
    elif a.precision == "bf16x3":
        x3_main(a.names or list(X3_CASES), a.rounds)
    else:
        tf32_main(a.names or list(CASES))
