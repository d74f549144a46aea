#!/usr/bin/env python
"""Measures the tensor-pipe roofline denominator for the MMA kind the convolutions use (tf32): cuBLAS fp32 GEMM with
TF32 tensor cores allowed, 8192^3, as a burst (best of 10, a kernel timed alone) and sustained (back to back for 4 s, a
kernel timed inside a long step) -- the same protocol MEASURED_PEAKS.json documents for its bf16 entry.  Also the
3xTF32-equivalent ceiling (one third of it) and the plain fp32 SIMT rate for context.
Prints one JSON line."""
import json
import time

import torch

dev = torch.device("cuda:0")
N = 8192
FLOP = 2.0 * N * N * N


def run(dtype, allow_tf32):
    torch.backends.cuda.matmul.allow_tf32 = allow_tf32
    a = torch.randn(N, N, device=dev, dtype=dtype)
    b = torch.randn(N, N, device=dev, dtype=dtype)
    c = torch.empty(N, N, device=dev, dtype=dtype)
    for _ in range(3):
        torch.matmul(a, b, out=c)
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(10):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.matmul(a, b, out=c)
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    # sustained: back to back for ~4 s
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 0
    t0 = time.time()
    e0.record()
    while time.time() - t0 < 4.0:
        for _ in range(20):
            torch.matmul(a, b, out=c)
        n += 20
        torch.cuda.synchronize()
    e1.record()
    torch.cuda.synchronize()
    sustained = e0.elapsed_time(e1) / n
    return FLOP / best / 1e9, FLOP / sustained / 1e9


tf32_burst, tf32_sus = run(torch.float32, True)
bf16_burst, bf16_sus = run(torch.bfloat16, True)
fp32_burst, fp32_sus = run(torch.float32, False)
print(json.dumps({"tf32_tflops": round(tf32_burst, 1), "tf32_tflops_sustained": round(tf32_sus, 1),
                  "bf16_tflops": round(bf16_burst, 1), "bf16_tflops_sustained": round(bf16_sus, 1),
                  "fp32_simt_tflops": round(fp32_burst, 1), "fp32_simt_tflops_sustained": round(fp32_sus, 1),
                  "how": "torch.matmul 8192^3 (cuBLAS), fp32 inputs with allow_tf32=True; best of 10 (burst) and back to "
                         "back for 4 s (sustained), CUDA events", "gpu": torch.cuda.get_device_name(0)}))
