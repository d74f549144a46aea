#!/usr/bin/env python
"""Single weight-gradient launches through the C ABI for timing.

    python tools/wgrad_probe.py [ns|mid|low|s2|t2] ...              tf32 kernel on the named shapes
    python tools/wgrad_probe.py --precision bf16x3 [name ...]       bf16x3 kernel on the 256^2 step's weight-gradient shapes

To compare two builds, run the tool in each checkout.
"""
import argparse
import os
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


def x3_main(names):
    """ms and algorithmic TFLOP/s of the bf16x3 weight gradient on the split planes of each named shape."""
    import torch
    from gif_b200 import ops
    from gif_b200._lib import lib
    dev = torch.device("cuda:0")
    ops.set_precision("bf16x3")
    print(f"{'shape':<14} {'ms':>8} {'TFLOP/s':>8}")
    for n in names:
        mode, b, r, ci, co, k = X3_CASES[n]
        mode = getattr(ops, mode)
        ho = ops.conv_out_size(r, k, mode)
        assert lib.gifb200_conv2d_wgrad_path(b, r, r, ci, ho, ho, co, k, mode, 3) == 3, n
        x = torch.randn(b, r, r, ci, device=dev)
        gy = torch.randn(b, ho, ho, co, device=dev)
        xp, gp = ops._planes(x), ops._planes(gy)                # split once: time the weight gradient alone
        ms = _time(lambda: ops._wgrad_raw(x, gy, k, mode, False, False, x_planes=xp))
        print(f"{n:<14} {ms:8.3f} {_tflops(mode, b, r, ci, co, k, ms):8.1f}", flush=True)
        del x, gy, xp, gp
        torch.cuda.empty_cache()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="tf32", choices=["tf32", "bf16x3"])
    ap.add_argument("names", nargs="*")
    a = ap.parse_args()
    if a.precision == "bf16x3":
        x3_main(a.names or list(X3_CASES))
    else:
        tf32_main(a.names or list(CASES))
