#!/usr/bin/env python
"""bench.py -- G+D training-step throughput (images/sec) at 256^2, batch 32 per GPU: BASELINE.json's metric on
configs[2] ("full G+D train step (R1 + path-length reg) 256x256 bs32, synthetic FFHQ + FLAME"), on H100 (sm_90a).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--no-ppl] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W

One JSON line on stdout (rank 0).  A "step" is one full iteration of the reference's loop body (train.py:80-252): D step
(real + fake forward, backward, Adam) + G step (G and D forward, backward, Adam, EMA), with the R1 penalty every 16th
iteration (train.py:145) and the path-length regulariser (adopted rule, PARITY UNPINNED) every iteration unless --no-ppl.
Inputs are synthetic FFHQ-shaped images U(-1,1), synthetic FLAME-render-shaped conditions U(-1,1), random identity indices;
weights are random-initialised as the reference's constructors do.

  value        images/sec, whole job, inputs resident in HBM, CUDA-event timed, max over ranks.
  e2e          same loop, but every step copies that step's inputs from PINNED HOST memory and reads the two loss
               scalars back (the call a user of train.py makes: host batch in, losses out).
  precision    --precision bf16x3 (default, the headline): the error-compensated tensor-core contraction, the mode that
               holds BASELINE.json's 1e-3 bar end to end (tests/test_models_gpu.py); the same step in plain tf32
               (faster, ~1e-3 forward / 1e-2 R1 deviation) is measured too and reported under "tf32_mode".
  roofline     the dominant kernel = the wgmma implicit-GEMM convolution (conv_tc_kernel): algorithmic FLOPs of
               every launch / its CUDA-event duration.  Peak: NVIDIA's H100 SXM data-sheet dense rates (700 W card):
               bf16x3 issues three bf16 MMAs per algorithmic MAC, so its ceiling is 989 TFLOP/s / 3; tf32: 495 TFLOP/s.
               A power-capped card runs lower clocks; "clocks" in the line records what the card ran at.
  cpu_baseline the REFERENCE ITSELF on the host cores: its unmodified train() (train.py:80-252) over its own model / loss
               modules (build-time extract oracle/_ref/pyref, oracle/ref_import.py), fp32, all usable threads, on a bounded
               sample: batch 1, one R1 iteration and one plain iteration combined with the loop's 1/16 R1 share (~1 min;
               the reference's CPU formulation needs ~25-50 s per image and iteration).  Falls back to the oracle port
               (kind "port") if the extract is absent.
  --impl reference   times only that CPU arm (plus a warm-up iteration), rank 0 only.
  extras       BASELINE.json configs[1] (generator forward 256^2 bs16) and configs[3] (FLAME-topology texture+normal
               rasterisation 256^2 bs64, forward and forward+backward, with its HBM roofline fraction).
  --dump-outputs DIR   the last timed step's losses and a seeded sample of the updated weights as DIR/<name>.npy
               (dump_outputs); inputs and weights are seeded, so two builds can be compared output for output.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

METRIC = "G+D train step images/sec @256x256 bs32/GPU"
RES, BATCH, VOCAB = 256, 32, 70_000
# NVIDIA H100 SXM data sheet (700 W): dense BF16 and TF32 tensor rates, HBM3 bandwidth
H100_BF16_TFLOPS, H100_TF32_TFLOPS, H100_HBM_GBS = 989.4, 494.7, 3350.0
DUMP_SAMPLE = 1 << 20


_REAL_STDOUT = None


def emit(line):
    data = (json.dumps(line) + "\n").encode()
    if _REAL_STDOUT is not None:
        os.write(_REAL_STDOUT, data)
    else:
        sys.stdout.write(data.decode())
        sys.stdout.flush()


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="gif_b200", choices=["gif_b200", "reference"])
    ap.add_argument("--no-ppl", action="store_true", help="drop the path-length regulariser from the G step")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-ppl-extra", action="store_true", help="skip the additional measurement without the PPL term")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--batch", type=int, default=BATCH)
    ap.add_argument("--texture-loss", action="store_true",
                    help="also time the step of the flagship reference run: no PPL, + texture-space interpolation loss")
    ap.add_argument("--no-graph", action="store_true", help="issue every kernel from Python instead of replaying CUDA graphs")
    ap.add_argument("--precision", default="bf16x3", choices=["tf32", "bf16x3"],
                    help="contraction mode of the tensor-core kernels for the HEADLINE numbers (gif_b200.ops.set_precision); "
                         "the other mode is measured as an extra")
    ap.add_argument("--no-other-precision", action="store_true", help="skip the extra measurement in the other precision mode")
    ap.add_argument("--no-extras", action="store_true", help="skip the configs[1] / configs[3] side measurements")
    ap.add_argument("--no-gpu-reference", action="store_true", help="skip timing the reference's own modules on this GPU (extra)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the losses and a seeded sample of the updated weights of the last timed step as DIR/<name>.npy")
    return ap.parse_args()


def dump_outputs(path, losses, trainer):
    """The result of the last timed step: the (d_loss, g_loss) pair train_iteration returns, and the weights that step left in
    the three networks -- all of them when small, else the same sample of positions on every run (a permutation seeded with 0 of
    the concatenated parameters, first DUMP_SAMPLE positions in ascending order; <= 13 MB in all)."""
    import numpy as np
    os.makedirs(path, exist_ok=True)
    np.save(os.path.join(path, "d_loss.npy"), np.array([float(losses[0])], dtype=np.float64))
    np.save(os.path.join(path, "g_loss.npy"), np.array([float(losses[1])], dtype=np.float64))
    for name, net in (("generator", trainer.generator), ("discriminator", trainer.discriminator), ("g_running", trainer.g_running)):
        flat = torch.cat([p.detach().reshape(-1).float() for p in net.parameters()])
        if flat.numel() > DUMP_SAMPLE:
            idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:DUMP_SAMPLE].sort().values
            flat = flat[idx.to(flat.device)]
        np.save(os.path.join(path, f"{name}_weights.npy"), flat.cpu().numpy().astype(np.float32))


# ------------------------------------------------------------------------------------------------ clocks
class ClockSampler:
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx.append(float(r[1]))
            except (ValueError, IndexError):
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# ------------------------------------------------------------------------------------------------ CPU arm
def usable_cores():
    """Host cores this process may really use: affinity mask, capped by the cgroup CPU quota (a 128-thread pool on a
    quota-limited container runs ~30x slower than a right-sized one) and by 32 (torch's conv kernels stop scaling)."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = min(n, max(1, int(float(quota) / float(period))))
    except (OSError, ValueError):
        pass
    return max(1, min(n, 32))


def cpu_arm(steps, warmup, budget_s=None):
    """The oracle port on the host cores: one D+G iteration at batch 1, 256^2 (no R1 / PPL) per step."""
    import golden_util as gu
    from oracle import stylegan2_oracle as O
    cores = usable_cores()
    torch.set_num_threads(cores)
    sdg = gu.seeded_state_dict(gu.g_shapes(100), 1)
    sdd = gu.seeded_state_dict(gu.d_shapes(RES), 3)
    gp = [k for k in sdg if "kernel" not in k and "embd" not in k]
    dp = [k for k in sdd if "kernel" not in k]
    for k in gp:
        sdg[k].requires_grad_(True)
    for k in dp:
        sdd[k].requires_grad_(True)
    b = 1
    cond, real, idx = gu.rand_uniform((b, 6, RES, RES), 1), gu.rand_uniform((b, 3, RES, RES), 2), gu.randint(100, (b,), 3)

    def one():
        with torch.no_grad():
            fake = O.generator_forward(cond, idx, sdg, 6)
        loss = O.d_logistic_loss(O.discriminator_forward(real, cond, sdd, RES), O.discriminator_forward(fake, cond, sdd, RES))
        torch.autograd.grad(loss, [sdd[k] for k in dp])
        fake = O.generator_forward(cond, idx, sdg, 6)
        gl = O.g_nonsat_loss(O.discriminator_forward(fake, cond, sdd, RES))
        torch.autograd.grad(gl, [sdg[k] for k in gp], allow_unused=True)

    t_all = time.perf_counter()
    for _ in range(warmup):
        one()
        if budget_s is not None and time.perf_counter() - t_all > budget_s / 4:
            break                                  # bounded: never spend more than a quarter of the budget warming up
    t0 = time.perf_counter()
    done = 0
    for _ in range(steps):
        one()
        done += 1
        if budget_s is not None and time.perf_counter() - t_all > budget_s:
            break                                  # bounded sample: the run must end within minutes whatever K is
    dt = (time.perf_counter() - t0) / max(done, 1)
    return {"value": b / dt, "unit": "images/sec", "cores": cores, "kind": "port", "steps_done": done,
            "sample": f"{done} iteration(s) of the D+G step at batch {b}, 256x256, no R1/PPL, oracle/stylegan2_oracle.py "
                      f"(torch CPU fp32, {cores} threads), {dt:.1f} s per iteration"}


def cpu_arm_reference(batch, warm_up, vocab=1000):
    """The reference's own loop and modules on the host cores (kind "reference"): iterations of the UNMODIFIED train() with the
    loop counter at [14 (warm-up, optional),] 15 (carries the R1 penalty, train.py:145) and 16 (plain).  Measured in the
    build container (8 cores): 49 s per plain iteration and 99 s per R1 iteration PER IMAGE -- the reference's grouped
    per-sample-weight convolutions and its conv2d-based upfirdn2d are ~25x slower on a CPU than the oracle port's
    modulate-input form -- hence batch 1 and two or three iterations: a bounded sample."""
    from oracle import ref_import, ref_train_runner
    if not ref_import.available():
        return None
    cores = usable_cores()
    torch.set_num_threads(cores)
    ref = ref_import.load()
    train = ref_import.load_train(with_gif_b200=False)
    kw = dict(embedding_vocab_size=vocab, rendered_flame_ascondition=True, normal_maps_as_cond=True, core_tensor_res=4, n_mlp=8)
    import contextlib
    with contextlib.redirect_stdout(None):
        G, Gr = ref.gen.StyledGenerator(**kw), ref.gen.StyledGenerator(**kw)
        D = ref.disc.Discriminator(size=RES, num_color_chnls=9, channel_multiplier=2)
    gen = torch.Generator().manual_seed(99)
    n = 3 if warm_up else 2
    batches = [(torch.rand(batch, 3, RES, RES, generator=gen) * 2 - 1, torch.rand(batch, 6, RES, RES, generator=gen) * 2 - 1,
                torch.randn(batch, 159, generator=gen), torch.randint(0, vocab, (batch,), generator=gen)) for _ in range(n)]
    stamps = []
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref_train_runner.run(train, G, D, Gr, batches, RES, vocab, first_i=14 if warm_up else 15, force_cpu=True, stamps=stamps)
    durs = [stamps[k + 1] - stamps[k] for k in range(n)]
    r1, plain = durs[-2], durs[-1]
    per_iter = (15 * plain + r1) / 16                       # the loop's R1 share (every 16th iteration)
    return {"value": batch / per_iter, "unit": "images/sec", "cores": cores, "kind": "reference", "steps_done": n,
            "s_per_iteration": {"plain": plain, "with_r1": r1, **({"warm_up": durs[0]} if warm_up else {})},
            "sample": f"the reference's unmodified train() (train.py:80-252) over its own model/ and loss modules, fp32 torch "
                      f"CPU, {cores} threads, batch {batch} at 256x256: {n} iterations ("
                      + (f"warm-up {durs[0]:.1f} s, " if warm_up else "") +
                      f"R1 iteration {r1:.1f} s, plain {plain:.1f} s) combined as (15 plain + 1 R1) / 16; no path-length term "
                      f"(the reference's own is unrunnable, SURVEY 8 L2)"}


def reference_on_gpu(batch=8, vocab=1000):
    """EXTRA, not the baseline of the contract: the reference's own modules and unmodified train() on THIS GPU through stock
    PyTorch / cuDNN (what a user of the reference gets on this GPU today), 1 warm-up + 2 timed plain iterations at a reduced
    batch (its per-sample weight tensors and unfused upfirdn2d make batch 32 slow to autotune).  torch's stock precision flags (cuDNN convolutions may use TF32, matmuls fp32)."""
    from oracle import ref_import, ref_train_runner
    if not ref_import.available() or not torch.cuda.is_available():
        return None
    import contextlib
    import warnings
    ref = ref_import.load()
    train = ref_import.load_train(with_gif_b200=False)
    kw = dict(embedding_vocab_size=vocab, rendered_flame_ascondition=True, normal_maps_as_cond=True, core_tensor_res=4, n_mlp=8)
    with contextlib.redirect_stdout(None):
        G, Gr = ref.gen.StyledGenerator(**kw), ref.gen.StyledGenerator(**kw)
        D = ref.disc.Discriminator(size=RES, num_color_chnls=9, channel_multiplier=2)
    gen = torch.Generator().manual_seed(98)
    batches = [(torch.rand(batch, 3, RES, RES, generator=gen) * 2 - 1, torch.rand(batch, 6, RES, RES, generator=gen) * 2 - 1,
                torch.randn(batch, 159, generator=gen), torch.randint(0, vocab, (batch,), generator=gen)) for _ in range(3)]
    stamps = []

    def sync(*_a):
        torch.cuda.synchronize()
        stamps.append(time.perf_counter())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref_train_runner.run(train, G, D, Gr, batches, RES, vocab, first_i=0, on_iteration_done=sync)
    per_iter = (stamps[2] - stamps[0]) / 2
    del G, D, Gr
    torch.cuda.empty_cache()
    return {"value": batch / per_iter, "unit": "images/sec", "batch": batch, "s_per_iteration": per_iter,
            "note": "the reference's unmodified train() over its own modules on this GPU (stock PyTorch ops / cuDNN, torch's default "
                    "precision flags: TF32 allowed in cuDNN convolutions), no R1 iteration in the sample; extra context, the contract's baseline is cpu_baseline"}


def cpu_baseline(batch, warm_up, port_budget_s):
    """The reference itself when its files are here (build-time extract / the container's tree), else the oracle port."""
    try:
        cb = cpu_arm_reference(batch, warm_up)
    except Exception as e:      # the baseline must never take the bench line down with it
        sys.stderr.write(f"reference CPU arm failed ({type(e).__name__}: {e}); falling back to the oracle port\n")
        cb = None
    return cb if cb is not None else cpu_arm(3, 1, budget_s=port_budget_s)


def reference_main(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    # the reference arm: batch 1, three iterations (warm-up, R1, plain) of the reference's own train(): ~2-3 minutes of CPU work
    cb = cpu_baseline(1, True, port_budget_s=180.0)
    line = {"impl": "reference", "metric": METRIC, "value": cb["value"], "unit": "images/sec", "n_gpus": args.gpus,
            "steps": cb["steps_done"], "warmup": args.warmup, "ms_per_step": 1000.0 / cb["value"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": "train_step_256_bs32: StyledGenerator + Discriminator(256, 9ch), D step + G step, Adam, EMA, R1 "
                                   "every 16th iteration (CPU arm: bounded sample at batch 1, see cpu_baseline.sample)"},
            "cpu_baseline": cb,
            "e2e": {"value": cb["value"], "unit": "images/sec", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    emit(line)


# ------------------------------------------------------------------------------------------------ GPU arm
def side_measurements(dev, trainer, resident):
    """BASELINE.json configs[1] and configs[3], measured in the driver-run bench so that they appear in the bench line."""
    from gif_b200 import rasterize
    from gif_b200.flame_synth import synthetic_flame_batch
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timeit(fn, iters=5, warm=3):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(iters):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return sorted(ts)[len(ts) // 2]
    out = {}
    # configs[1]: StyledGenerator forward 256^2 bs16 (105.3 GFLOP / image, SURVEY 8d)
    G = trainer.g_running
    cond, idx = resident[0][1][:16], resident[0][2][:16]
    with torch.no_grad():
        ms = timeit(lambda: G(cond, step=6, input_indices=idx))
    out["config1_generator_fwd_256_bs16"] = {"images_per_s": 16 / ms * 1e3, "ms": ms, "tflops_algorithmic": 16 * 105.3 / ms}
    # configs[3]: FLAME-topology texture + normal rasterisation 256^2 bs64 (one pass, two attribute sets), fwd and fwd+bwd
    b, h, w = 64, 256, 256
    fv, fc = synthetic_flame_batch(b, h, w, seed=0, device=dev)
    F = fv.shape[1]
    nrm = torch.rand_like(fc)
    fvg, fcg, ng = fv.clone().requires_grad_(True), fc.clone().requires_grad_(True), nrm.clone().requires_grad_(True)
    g1 = torch.randn(b, h, w, 3, device=dev)

    def fwd_bwd():
        _, _, im, nm = rasterize.rasterize(fvg, h, w, fcg, ng)
        torch.autograd.backward([im, nm], [g1, g1])
    ms_f = timeit(lambda: rasterize.rasterize(fv, h, w, fc, nrm))
    ms_fb = timeit(fwd_bwd)
    fwd_bytes = 3 * F * 36 + h * w * (4 + 4 + 12 + 12)                  # SURVEY 8d, texture+normal: 3.96 MB / image
    bwd_bytes = h * w * (12 + 12 + 4) + 3 * F * 36 + 3 * F * 36
    hbm = H100_HBM_GBS
    out["config3_rasterize_texture_normal_256_bs64"] = {
        "renders_per_s_fwd": b / ms_f * 1e3, "renders_per_s_fwd_bwd": b / ms_fb * 1e3, "fwd_ms": ms_f, "fwd_bwd_ms": ms_fb,
        "roofline": {"bound": "hbm", "achieved": b * fwd_bytes / ms_f / 1e6, "peak": hbm, "unit": "GB/s",
                     "frac": b * fwd_bytes / ms_f / 1e6 / hbm, "frac_fwd_bwd": b * (fwd_bytes + bwd_bytes) / ms_fb / 1e6 / hbm,
                     "algorithmic_bytes_per_image": {"fwd": fwd_bytes, "bwd": bwd_bytes}}}
    return out


def main():
    args = parse()
    # Libraries (NCCL prints its version banner) write to stdout: keep fd 1 for the ONE JSON line, send the rest to stderr.
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)
    if args.impl == "reference":
        return reference_main(args)
    from gif_b200 import _lib, ops
    from gif_b200.distributed import broadcast_module, init_from_env
    from gif_b200.train_step import GifTrainer
    from gif_b200 import losses as losses_mod
    import torch.distributed as dist

    rank, world, local = init_from_env("nccl")
    assert world == args.gpus or world == 1, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    assert torch.cuda.is_available(), "bench.py needs a GPU (there is no CPU fallback for the product path)"
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    ops.set_precision(args.precision)
    B = args.batch
    trainer = GifTrainer(dev, RES, VOCAB, r1_every=16, ppl=not args.no_ppl, world_size=world, seed=0)
    broadcast_module(trainer.generator)
    broadcast_module(trainer.discriminator)
    trainer.g_running.load_state_dict(trainer.generator.state_dict())

    gen = torch.Generator().manual_seed(1234 + rank)
    n_host = 4   # distinct pinned host batches cycled through (each 75.5 MB)
    host = [(torch.rand(B, 3, RES, RES, generator=gen).mul_(2).sub_(1).pin_memory(),
             torch.rand(B, 6, RES, RES, generator=gen).mul_(2).sub_(1).pin_memory(),
             torch.randint(0, VOCAB, (B,), generator=gen).pin_memory()) for _ in range(n_host)]
    resident = [tuple(t.to(dev) for t in hb) for hb in host]
    # FLAME labels [shape 100 | exp 50 | pose 6 | cam 3] for the optional texture-interpolation term (random FLAME params)
    flm = torch.cat([torch.randn(B, 150, generator=gen), (torch.rand(B, 6, generator=gen) * 2 - 1) * torch.tensor([0.2, 0.5, 0.1, 0.3, 0.02, 0.02]),
                     torch.rand(B, 1, generator=gen) * 3 + 7, (torch.rand(B, 2, generator=gen) * 2 - 1) * 0.02], 1).to(dev)
    h2d = sum(t.numel() * t.element_size() for t in host[0])
    # R1 must fall inside every timed window: start the iteration counter so that the window contains
    # ceil(K/16) penalty iterations, the same share as in the reference's loop.
    last = [None]

    def run(n, e2e):
        out = None
        for s in range(n):
            if e2e:
                hb = host[s % n_host]
                if trainer._graphs is not None:
                    real, cond, idx = hb           # copied from pinned host memory straight into the graphs' input buffers
                else:
                    real, cond, idx = (t.to(dev, non_blocking=True) for t in hb)
            else:
                real, cond, idx = resident[s % n_host]
            out = trainer.train_iteration(real, cond, idx, flm if trainer.interp_tex_loss is not None else None)
            if e2e:
                out = (out[0].item(), out[1].item())      # device -> host read of the step's result
        last[0] = out
        return out

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(n, e2e):
        trainer.iteration = 16 - 1 - (n - 1) % 16 if n < 16 else 0      # the last iteration of a short window is an R1 one
        if os.environ.get("GIFB200_TIMED_FIRST_ITERATION"):              # profiling only: e.g. 0 = a window of plain iterations
            trainer.iteration = int(os.environ["GIFB200_TIMED_FIRST_ITERATION"])
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(n, e2e)
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms)

    # warm-up (also includes one R1 iteration so that every kernel variant is loaded)
    trainer.iteration = 16 - args.warmup
    run(args.warmup, False)
    barrier()
    graph_note = "off (--no-graph)"
    if not args.no_graph:
        try:
            trainer.capture(B, RES)
            trainer.iteration = 14
            run(2, False)                      # one replay of each graph before timing
            barrier()
            graph_note = "3 CUDA graphs per iteration (cut at the two gradient all-reduces) x 2 variants (with / without R1), replayed"
        except Exception as e:                 # capture is an optimisation of the launch path, never a different compute path
            trainer._graphs = None
            graph_note = f"capture failed, eager launches: {type(e).__name__}: {str(e)[:200]}"
            torch.cuda.synchronize()

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    launches0 = _lib.launch_count()
    trainer.replayed_launches = 0
    use_graph = trainer._graphs is not None
    ops.PROFILE = [] if (rank == 0 and not use_graph) else None
    cuprof = bool(os.environ.get("GIFB200_CUPROFILE"))   # `ncu --profile-from-start off`: capture exactly the timed steps
    if cuprof:
        torch.cuda.profiler.start()
    ms = timed(args.steps, False)
    if cuprof:
        torch.cuda.profiler.stop()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last[0], trainer)
    launches = _lib.launch_count() - launches0 + trainer.replayed_launches
    prof = ops.PROFILE
    ops.PROFILE = None
    clocks = sampler.stop() if rank == 0 else None
    prof_note = "per-launch CUDA events inside the timed region"
    if use_graph:
        # graph replays cannot carry per-launch events: time the same kernels in a separate eager pass of the same steps
        # (all ranks run it -- it contains the gradient all-reduces -- only rank 0 records events)
        # the captured graphs' private memory pools and an eager iteration's activations do not fit in 80 GB together:
        # release the graphs for this pass and capture them again afterwards
        trainer._graphs = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        ops.PROFILE = [] if rank == 0 else None
        timed(min(args.steps, 4), False)
        prof = ops.PROFILE
        ops.PROFILE = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        trainer.capture(B, RES)
        trainer.iteration = 14
        run(2, False)
        barrier()
        prof_note = ("per-launch CUDA events in a separate eager pass of %d steps after the timed region (CUDA-graph replays "
                     "cannot carry events; same kernels, same shapes)" % min(args.steps, 4))
    value = world * B * args.steps / (ms / 1000.0)

    e2e = None
    if not args.no_e2e:
        ms_e = timed(args.steps, True)
        e2e = {"value": world * B * args.steps / (ms_e / 1000.0), "unit": "images/sec", "h2d_bytes_per_step": h2d * world,
               "d2h_bytes_per_step": 8 * world}

    extra_no_ppl = None
    if trainer.ppl is not None and not args.no_ppl_extra:
        # the same step without the (parity-unpinned, never enabled in a shipped reference config) path-length regulariser
        trainer.ppl = None
        trainer._graphs = None
        try:
            if not args.no_graph:
                trainer.capture(B, RES)
                trainer.iteration = 14
                run(2, False)
            else:
                trainer.iteration = 13
                run(3, False)
            ms_np = timed(args.steps, False)
            extra_no_ppl = {"value": world * B * args.steps / (ms_np / 1000.0), "unit": "images/sec",
                            "ms_per_step": ms_np / args.steps}
        except Exception as e:
            extra_no_ppl = {"error": f"{type(e).__name__}: {str(e)[:160]}"}
    extra_tex = None
    if args.texture_loss:
        # the flagship reference configuration (configurations.py:217, run 29): no PPL, + the texture-space interpolation
        # loss of train.py:224-238 (31 interpolated FLAME parameter sets -> condition renders -> one more generator
        # forward/backward -> texture stealing -> pairwise loss), FLAME model data synthetic
        trainer.ppl = None
        trainer._graphs = None
        try:
            trainer.interp_tex_loss = trainer._build_texture_loss(dev, B)
            trainer.iteration = 13
            run(3, False)
            if not args.no_graph:
                trainer.capture(B, RES)
                trainer.iteration = 14
                run(2, False)
            ms_t = timed(args.steps, False)
            extra_tex = {"value": world * B * args.steps / (ms_t / 1000.0), "unit": "images/sec", "ms_per_step": ms_t / args.steps}
        except Exception as e:
            extra_tex = {"error": f"{type(e).__name__}: {str(e)[:200]}"}
        trainer.interp_tex_loss = None
    other_mode = None
    if not args.no_other_precision:
        # the same step (same flags as the headline line: with the path-length term unless --no-ppl) in the other mode
        other = "tf32" if args.precision == "bf16x3" else "bf16x3"
        ops.set_precision(other)
        saved_ppl = trainer.ppl
        trainer.ppl = None if args.no_ppl else losses_mod.PathLengthRegularizor()
        trainer._graphs = None
        try:
            trainer.iteration = 13
            run(3, False)
            if not args.no_graph:
                trainer.capture(B, RES)
                trainer.iteration = 14
                run(2, False)
            ms_o = timed(args.steps, False)
            other_mode = {"precision": other, "value": world * B * args.steps / (ms_o / 1000.0), "unit": "images/sec",
                          "ms_per_step": ms_o / args.steps}
            if trainer.ppl is not None:
                trainer.ppl = None
                trainer._graphs = None
                if not args.no_graph:
                    trainer.capture(B, RES)
                    trainer.iteration = 14
                    run(2, False)
                else:
                    trainer.iteration = 13
                    run(3, False)
                ms_o2 = timed(args.steps, False)
                other_mode["same_step_without_path_length_reg"] = {"value": world * B * args.steps / (ms_o2 / 1000.0),
                                                                   "ms_per_step": ms_o2 / args.steps}
        except Exception as e:
            other_mode = {"precision": other, "error": f"{type(e).__name__}: {str(e)[:200]}"}
        trainer.ppl = saved_ppl
        trainer._graphs = None
        ops.set_precision(args.precision)
    extras = None
    if rank == 0 and not args.no_extras:
        try:
            extras = side_measurements(dev, trainer, resident)
        except Exception as e:
            extras = {"error": f"{type(e).__name__}: {str(e)[:200]}"}
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    # ---- roofline of the dominant kernel from the per-launch CUDA events recorded inside the timed region
    roof = None
    if prof:
        torch.cuda.synchronize()
        shapes = {}
        for a, b, f, tag, key in prof:
            e = shapes.setdefault(key, [0, 0.0, 0.0])
            e[0] += 1; e[1] += a.elapsed_time(b); e[2] += f
        if os.environ.get("GIFB200_SHAPE_PROFILE"):
            with open(os.environ["GIFB200_SHAPE_PROFILE"], "w") as fh:
                for key, (n, t, f) in sorted(shapes.items(), key=lambda kv: -kv[1][1]):
                    fh.write(f"{key}  launches={n}  ms={t:.3f}  TFLOP/s={f / (t * 1e-3) / 1e12 if t > 0 else 0:.1f}\n")
        prof = [(a, b, f, tag) for a, b, f, tag, key in prof if key[0] == "conv"]
        tot_ms = sum(a.elapsed_time(b) for a, b, _, _ in prof)
        tot_fl = sum(f for _, _, f, _ in prof)
        prof_steps = min(args.steps, 4) if use_graph else args.steps
        if args.precision == "bf16x3":
            # three bf16 MMAs per algorithmic multiply-add: the ceiling for ALGORITHMIC flops is the bf16 peak / 3
            peak = H100_BF16_TFLOPS / 3
            peak_src = ("H100 SXM data sheet, dense BF16 989 TFLOP/s at 700 W, / 3 (bf16x3 issues hi*hi + hi*lo + lo*hi: three "
                        "bf16 MMAs per algorithmic multiply-add)")
        else:
            peak = H100_TF32_TFLOPS
            peak_src = "H100 SXM data sheet, dense TF32 495 TFLOP/s at 700 W"
        ach_all = tot_fl / (tot_ms * 1e-3) / 1e12 if tot_ms > 0 else 0.0
        ns = [(a.elapsed_time(b), f) for a, b, f, tag in prof if tag == "northstar"]
        # dominant kernel instance: conv_tc_kernel<128> on the north-star layer (B,128,256,256)->128, 3x3:
        # algorithmic FLOPs per launch = 2*9*128*128 per output pixel * 32*256*256 pixels = 618.5 GFLOP
        ach = (sum(f for _, f in ns) / (sum(t for t, _ in ns) * 1e-3) / 1e12) if ns else ach_all
        kname = ("conv_tc_kernel<128, X3> (wgmma bf16, bf16x3 error-compensated implicit GEMM)" if args.precision == "bf16x3"
                 else "conv_tc_kernel<128> (wgmma tf32 implicit GEMM)")
        roof = {"bound": "tensor", "kernel": kname + " on the north-star layer ModulatedConv2d 128->128 3x3 @256x256, batch 32",
                "achieved": ach, "peak": peak, "unit": "TFLOP/s", "frac": ach / peak,
                "algorithmic_flops_per_launch": 2.0 * 9 * 128 * 128 * 32 * 256 * 256,
                "algorithmic_hbm_bytes_per_launch": 2 * 32 * 256 * 256 * 128 * 4 + 9 * 128 * 128 * 4,
                "launches_of_this_shape": len(ns), "avg_launch_ms": (sum(t for t, _ in ns) / len(ns)) if ns else None,
                "all_tensor_core_conv_launches": {"achieved": ach_all, "frac": ach_all / peak},
                "peak_source": peak_src,
                "executed_mma_tflops": ach * (3 if args.precision == "bf16x3" else 1),
                "launches": len(prof), "kernel_ms_per_step": tot_ms / prof_steps,
                "share_of_step": (tot_ms / prof_steps) / (ms / args.steps), "measured": prof_note}
    ref_gpu = None
    if not args.no_gpu_reference and world == 1:
        try:
            trainer._graphs = None
            torch.cuda.empty_cache()
            ref_gpu = reference_on_gpu()
        except Exception as e:
            ref_gpu = {"error": f"{type(e).__name__}: {str(e)[:200]}"}
    cb = None
    if not args.no_cpu_baseline and world == 1:      # the CPU baseline is a rank-0, N=1 measurement
        cb = cpu_baseline(1, False, port_budget_s=40.0)   # the reference's own train() at batch 1: an R1 and a plain iteration
    line = {"metric": METRIC, "value": value, "unit": "images/sec", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None,
            "dtype": ("bf16x3 error-compensated tensor-core contraction (two-term bf16 operands, 3 MMAs per slice), f32 accumulate/storage"
                      if args.precision == "bf16x3" else "tf32 tensor-core contraction, f32 accumulate/storage"),
            "precision": args.precision, "data": "synthetic",
            "config": {"workload": "train_step_256_bs32: StyledGenerator(70000 ids) + Discriminator(256, 9ch), D step + G step, "
                                   "Adam, EMA, R1 every 16th iteration" + ("" if args.no_ppl else ", path-length reg every iteration"),
                       "global_batch": B * world, "resolution": RES, "parallelism": f"dp{world}", "cuda_graph": graph_note,
                       "l2_policy": "inputs (4 x 75.5 MB batches, 1+ GB activations per layer) exceed the 50 MB L2"},
            "clocks": clocks, "gpu_launches": launches, "e2e": e2e, "roofline": roof, "cpu_baseline": cb,
            "same_step_without_path_length_reg": extra_no_ppl,
            ("tf32_mode" if args.precision == "bf16x3" else "bf16x3_mode"): other_mode,
            "other_configs": extras, "reference_modules_on_this_gpu": ref_gpu,
            "same_step_with_texture_interpolation_loss_instead_of_ppl": extra_tex}
    emit(line)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
