"""One-process-per-GPU data parallelism: replaces train.py's nn.DataParallel (train.py:344,356,358).

The reference re-broadcasts every parameter on each of its 5 wrapped forwards per iteration and reduces gradients to
GPU 0.  Here every rank holds full replicas (G, D, EMA-G, Adam state), draws its own batch, and after each
``backward()`` the gradients of the net being optimised are averaged with ONE collective per net on a pre-flattened fp32
buffer (``torch.distributed`` all-reduce: NCCL over NVLink 5 / NVSwitch on GPUs, gloo in the CPU tests).  Replicas stay
bit-identical because they apply identical averaged gradients (SURVEY 8e).  Minibatch-stddev groups stay inside a rank
(per-rank batch % 4 == 0), the rasteriser is per-sample: no other exchange exists on the path.

A plain DistributedDataParallel wrapper does not fit the reference's loop (requires_grad toggling per phase,
``autograd.grad`` for R1, two forwards per backward, parameters of unused resolutions), hence the explicit buffer.
"""
import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """Initialise torch.distributed from torchrun's environment; returns (rank, world_size, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, rank=rank, world_size=world, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend, rank=rank, world_size=world)
    return rank, world, local


class FlatGradAllReducer:
    """Gradient exchange for one network: a flat fp32 buffer with one slot per parameter that can receive a gradient.

    Per step: ``zero()`` clears every ``.grad`` (sets it to None -- no memset, and autograd then MOVES each freshly computed
    gradient into ``.grad`` instead of launching one ``grad += new`` kernel per parameter: ~500 launches and two full
    read-modify-write passes over the gradients per iteration in round 1); ``all_reduce_sum()`` packs the gradients into
    the flat buffer with one multi-tensor copy, runs ONE collective (or a few contiguous buckets, issued back to back),
    and points every ``.grad`` at its slot.  With one rank nothing is packed at all: the optimiser reads the gradients
    where autograd left them, and parameters that were not used keep ``grad = None`` exactly as in the reference.
    ``pre_scale()`` is the 1/world factor to fold into the loss so that the SUM already yields the mean."""

    def __init__(self, params, world_size=None, group=None, bucket_bytes=None):
        self.params = [p for p in params]
        self.group = group
        self.world = world_size if world_size is not None else (dist.get_world_size(group) if dist.is_initialized() else 1)
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device if self.params else torch.device("cpu")
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        self.views = []
        o = 0
        for p in self.params:
            self.views.append(self.flat[o:o + p.numel()].view_as(p))
            o += p.numel()
        self.nbytes = n * 4
        per = n if not bucket_bytes else max(1, int(bucket_bytes) // 4)
        self.buckets = [self.flat[a:min(a + per, n)] for a in range(0, max(n, 1), per)] if n else []
        self._dirty = [False] * len(self.params)

    def attach(self):
        """Make every parameter's .grad a view into the (zeroed) flat buffer: backward then accumulates straight into it.
        The round-1 scheme; kept for callers that want in-place accumulation across several backward calls."""
        self.flat.zero_()
        self._dirty = [True] * len(self.params)
        for p, v in zip(self.params, self.views):
            p.grad = v

    def zero(self):
        for p in self.params:
            p.grad = None

    def pre_scale(self):
        """Factor to multiply the local loss by so that ``all_reduce_sum()`` leaves the MEAN gradient in the buffer."""
        return 1.0 / self.world

    def pack(self):
        """Gather the gradients autograd produced into their slots (one multi-tensor copy) and point every ``.grad`` at its
        slot; parameters without a gradient on this rank contribute zeros (another rank may have used them); gradients
        that already live in their slot (after ``attach()``) are left alone.  Stream-ordered device work only, so it can
        be the tail of a captured CUDA graph (the collective itself stays outside).  A no-op with a single rank."""
        if self.world <= 1:
            return
        src, dst = [], []
        for i, (p, v) in enumerate(zip(self.params, self.views)):
            g = p.grad
            if g is None:
                if self._dirty[i]:                       # slots start zeroed and stay zero until a gradient is copied in
                    v.zero_()
                    self._dirty[i] = False
            elif g.data_ptr() != v.data_ptr():
                src.append(g)
                dst.append(v)
                self._dirty[i] = True
        if src:
            torch._foreach_copy_(dst, src)
        for p, v in zip(self.params, self.views):
            p.grad = v

    def reduce(self):
        """The collective on the packed buffer: SUM over ranks, in place (bucketed).  A no-op with a single rank."""
        if self.world <= 1:
            return
        works = [dist.all_reduce(b, op=dist.ReduceOp.SUM, group=self.group, async_op=True) for b in self.buckets]
        for w in works:
            w.wait()

    def all_reduce_sum(self):
        """pack() + reduce().  Use with a loss pre-scaled by ``pre_scale()``."""
        self.pack()
        self.reduce()

    def all_reduce_mean(self):
        """SUM over ranks then 1/world (for losses that were not pre-scaled)."""
        self.all_reduce_sum()
        if self.world > 1:
            self.flat.mul_(1.0 / self.world)


class DataParallel(torch.nn.Module):
    """Stand-in for ``torch.nn.DataParallel`` in the reference's train.py (:344, :356, :358, :367): exposes ``.module``
    (so ``generator.module.get_embddings()``, ``generator.module.parameters()``, ``generator.module.z_to_w`` and the
    ``module.``-prefixed checkpoint keys keep working), runs ``forward`` on the LOCAL replica only -- one process per GPU
    replaces the reference's one-process scatter/replicate/gather -- and leaves the gradient exchange to the optimiser
    hook below.  ``device_ids`` / ``output_device`` / ``dim`` are accepted and ignored."""

    def __init__(self, module, device_ids=None, output_device=None, dim=0):
        super().__init__()
        self.module = module

    def forward(self, *inputs, **kwargs):
        return self.module(*inputs, **kwargs)


_reducers = {}
_hook_handle = None


def _optimizer_pre_step_hook(optimizer, args, kwargs):
    """Runs before EVERY ``optimizer.step()`` of the process once installed: averages the gradients of that optimiser's
    parameters across ranks through a cached FlatGradAllReducer (train.py calls ``loss.backward(); optimizer.step()`` and
    knows nothing about ranks).  Parameters without a gradient contribute zeros on this rank (another rank may have used
    them)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return None
    red = _reducers.get(id(optimizer))
    params = [p for g in optimizer.param_groups for p in g["params"]]
    if red is None or len(red.params) != len(params) or any(a is not b for a, b in zip(red.params, params)):
        red = FlatGradAllReducer(params, dist.get_world_size())
        _reducers[id(optimizer)] = red
    # parameters without a gradient here (e.g. the unused high-resolution blocks, gen.py:175) contribute zeros; Adam's
    # update for an all-zero gradient is exactly 0 (0 / (0 + eps))
    red.all_reduce_mean()
    return None


def install_data_parallel_shim():
    """``torch.nn.DataParallel = gif_b200.distributed.DataParallel`` + the global optimiser pre-step hook.  Called by
    ``gif_b200.install_as_reference_modules()`` so that the reference's train.py runs unchanged under
    ``torchrun --nproc-per-node N train.py ...`` (one process per GPU, NCCL all-reduce instead of DataParallel's
    scatter/gather).  Idempotent.  Returns the original class so a caller can restore it."""
    global _hook_handle
    original = getattr(torch.nn, "_gifb200_original_DataParallel", None) or torch.nn.DataParallel
    torch.nn._gifb200_original_DataParallel = original
    torch.nn.DataParallel = DataParallel
    torch.nn.parallel.DataParallel = DataParallel
    if _hook_handle is None:
        from torch.optim.optimizer import register_optimizer_step_pre_hook
        _hook_handle = register_optimizer_step_pre_hook(_optimizer_pre_step_hook)
    return original


def uninstall_data_parallel_shim():
    global _hook_handle
    original = getattr(torch.nn, "_gifb200_original_DataParallel", None)
    if original is not None:
        torch.nn.DataParallel = original
        torch.nn.parallel.DataParallel = original
    if _hook_handle is not None:
        _hook_handle.remove()
        _hook_handle = None
    _reducers.clear()


def broadcast_module(module, src=0):
    """Make all replicas start from rank `src`'s parameters and buffers."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return
    ts = list(module.parameters()) + list(module.buffers())
    with torch.no_grad():
        for t in ts:
            dist.broadcast(t, src)
    # the collective writes in place without bumping the version counters (which the prepared-weight cache keys on)
    torch.autograd.graph.increment_version(ts)
