"""torch.autograd wrappers over the C ABI (include/gifb200.h).

Conventions
  * activations are fp32 CUDA tensors in channels-last *physical* layout, shape (B, H, W, C), contiguous
    ("NHWC"); the module classes in gif_b200/model convert from/to the reference's NCHW view at the boundary
    (a zero-copy permute when the tensor came from one of these ops);
  * every Function's ``backward`` is written in terms of other Functions of this file, so arbitrary-order
    derivatives exist (R1 needs the double backward of every discriminator op, losses.py:91; the path-length
    regulariser needs it for every generator op);
  * there is no CPU / eager fallback: non-CUDA tensors raise.
"""
import math
import weakref

import torch

from ._lib import GifB200Error, check, lib, ptr, require_cuda, stream

S1, S2, T2 = 0, 1, 2          # conv modes of gifb200_conv2d
_ADJ_MODE = {S1: S1, S2: T2, T2: S2}
CONV_IMPL = 0                 # 0 auto, 1 force SIMT fp32, 2 force the tensor-core path (tests flip this)
WGRAD_IMPL = 0                # same for the weight-gradient kernel
_PRECISION = "tf32"


_WEIGHT_GRADS = [True]


class input_gradient_only:
    """``with ops.input_gradient_only():`` around a ``torch.autograd.grad(..., inputs=<activations / latents>)`` call: a custom
    Function's ``ctx.needs_input_grad`` says which inputs REQUIRE grad, not which gradients this particular call asks for, so
    the R1 penalty (gradient w.r.t. the image) and the path-length term (gradient w.r.t. w) would compute -- and autograd would
    throw away -- the weight gradient of every convolution on the way: a third of the tensor work of that pass.  Inside the
    block the convolution Functions skip their weight gradients, the tails skip their bias and noise-branch gradients (side
    branches that end in parameters or in the condition receive NO gradient: ask only for gradients w.r.t. the image / the
    latent chain), and the StyledConv tail / modulation backwards are recorded as single nodes with a fused second-order
    kernel (``_TailBwdCG``)."""

    def __enter__(self):
        self.prev = _WEIGHT_GRADS[0]
        _WEIGHT_GRADS[0] = False

    def __exit__(self, *a):
        _WEIGHT_GRADS[0] = self.prev
        return False


def set_precision(mode):
    """"tf32":   convolutions that qualify run on the tensor cores (tf32, fp32 accumulate) and their operand producers round
                 to tf32 (~3e-4 per operator);
    "bf16x3": the same kernels in their error-compensated mode -- operands split into two bf16 terms
                 (gifb200_split_bf16), three bf16 MMAs per slice, fp32 accumulate: ~1e-5 per operator at 1.5x the
                 tensor work; the mode that holds BASELINE.json's 1e-3 bar END TO END (G, D, R1);
    "fp32":   every convolution runs on the exact-fp32 SIMT kernels (parity arbitration, odd shapes)."""
    global CONV_IMPL, _PRECISION
    if mode not in ("tf32", "bf16x3", "fp32"):
        raise ValueError(mode)
    _PRECISION = mode
    CONV_IMPL = {"tf32": 0, "bf16x3": 3, "fp32": 1}[mode]


def get_precision():
    return _PRECISION


def tf32_enabled():
    """True when operand producers should round their outputs to tf32 (tf32 consumers truncate)."""
    return _PRECISION == "tf32" and CONV_IMPL != 1


def tc_enabled():
    """True when convolutions run on the tensor cores (tf32 or bf16x3): layers zero-pad odd channel counts to 32."""
    return _PRECISION in ("tf32", "bf16x3") and CONV_IMPL != 1


def _planes(x):
    """The two-term bf16 expansion of an fp32 tensor (operand format of the bf16x3 contraction), cached on the tensor
    object under its version counter: the forward convolution, the weight gradient (x) and the input gradient + weight
    gradient (gy) each reuse one split pass."""
    c = getattr(x, "_gifb200_planes", None)
    if c is not None and c[0] == x._version:
        return c[1]
    B, C = x.shape[0], x.shape[-1]
    P = x.numel() // max(B * C, 1)
    pl = torch.empty((2,) + tuple(x.shape), dtype=torch.bfloat16, device=x.device)
    check(lib.gifb200_split_bf16(ptr(x), None, ptr(pl), B, P, C, stream()), "gifb200_split_bf16")
    x._gifb200_planes = (x._version, pl)
    return pl


def _carry_planes(x, planes):
    if planes is not None:
        x._gifb200_planes = (x._version, planes)


def _tag(t, rounded):
    """Marks a tensor whose values are exactly representable in tf32 (so a tensor-core consumer needs no rounding pass).
    The mark records the tensor's version counter: autograd's in-place gradient accumulation (``buffer += grad``) keeps the
    Python object -- and its attributes -- but bumps the version, which invalidates the mark."""
    if rounded:
        t._gifb200_tf32 = t._version
    return t


def _is_tf32(t):
    return getattr(t, "_gifb200_tf32", None) == t._version


def _round_tf32_raw(x):
    y = torch.empty_like(x)
    check(lib.gifb200_axpby(ptr(x), None, ptr(y), x.numel(), 1.0, 0.0, 1, stream()), "gifb200_axpby(round)")
    return y


def _tc_operand(x, path, planes=None):
    """What a convolution kernel on ``path`` reads for the fp32 operand x: 3 (bf16x3) its split planes (``planes`` when the
    caller already has them); 2 (tf32) x when it is marked tf32-representable, else a rounded and marked copy (the tensor
    cores truncate, see gifb200.h); any other path (exact fp32 SIMT) x itself."""
    if path == 3:
        return planes if planes is not None else _planes(x)
    if path == 2 and not _is_tf32(x):
        return _tag(_round_tf32_raw(x), True)
    return x


PROFILE = None   # bench.py sets this to a list; every tensor-core conv launch then appends (ev0, ev1, flops, tag, key)


def _profiled(on, launch, tag, key, out_hw):
    """Runs ``launch()``.  When PROFILE is a list and ``on``, the launch is bracketed by CUDA events and PROFILE receives
    (ev0, ev1, algorithmic flops, tag, key), key = (kind, mode, B, Hi, Wi, Ci, Co, k)."""
    if PROFILE is None or not on:
        launch()
        return
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    launch()
    ev1.record()
    _, mode, B, Hi, Wi, Ci, Co, k = key
    pix = Hi * Wi if mode == T2 else out_hw[0] * out_hw[1]          # algorithmic MACs: taps * Ci * Co per site
    PROFILE.append((ev0, ev1, 2.0 * B * pix * Ci * Co * k * k, tag, key))


_ws_cache = {}
_ws_retired = []


def _workspace(nbytes, device):
    """A per-(device, stream) scratch buffer, grown on demand (stream-ordered reuse: all our launches are on the current
    stream).  A superseded buffer is retired, never freed: a captured CUDA graph may hold its address."""
    if nbytes == 0:
        return None
    key = (device.index, torch.cuda.current_stream().cuda_stream)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        if buf is not None:
            _ws_retired.append(buf)
        buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


# --------------------------------------------------------------------------------------------- convolution
def conv_out_size(hi, k, mode):
    if mode == S1:
        return hi
    if mode == S2:
        return (hi - k) // 2 + 1
    return 2 * (hi - 1) + k


def _conv_raw(x, w, k, mode, flip, transposed, out_hw, epilogue=None, planes=None):
    """epilogue: None (plain accumulator) or (bias_flat or None, slope, gain, round_tf32) fused into the kernel.
    planes: the bf16x3 operand of the INPUT when the caller already has it (x then only supplies shape and device)."""
    require_cuda(x, w)
    B, Hi, Wi, Ci = x.shape
    T, R, S = w.shape
    Co = R if not transposed else S
    assert T == k * k and (S if not transposed else R) == Ci, f"weight {tuple(w.shape)} vs input channels {Ci}"
    Ho, Wo = out_hw
    y = torch.empty((B, Ho, Wo, Co), dtype=torch.float32, device=x.device)
    nws = lib.gifb200_conv2d_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, int(transposed), CONV_IMPL)
    path = 1 if nws == 0 else (3 if CONV_IMPL == 3 else 2)
    impl = 1 if CONV_IMPL == 3 and path == 1 else CONV_IMPL     # shape outside the tensor-core path: exact fp32 SIMT
    xin = _tc_operand(x, path, planes)
    if path == 2:
        x = xin
    ws, staged = _staged_workspace(w, nws, flip, transposed, impl, (Ci, Co, k), x.device)
    if staged:
        impl |= 0x10                             # GIFB200_CONV_PRESTAGED: skip the staging pass
    if epilogue is None:
        act, bias, slope, gain, rt = 0, None, 1.0, 1.0, 0
    else:
        bias, slope, gain, rt = epilogue
        act = 1
    tag = "northstar" if (mode == S1 and Ci == 128 and Co == 128 and Ho == 256 and k == 3) else ""
    _profiled(nws > 0, lambda: check(lib.gifb200_conv2d(ptr(xin), ptr(w), ptr(y), B, Hi, Wi, Ci, Ho, Wo, Co, k, mode,
                                                        int(flip), int(transposed), impl, act, ptr(bias), float(slope),
                                                        float(gain), int(rt), ptr(ws), nws, stream()), "gifb200_conv2d"),
              tag, ("conv", mode, B, Hi, Wi, Ci, Co, k), out_hw)
    return y, x


def _wgrad_raw(x, gy, k, mode, flip, transposed, x_planes=None):
    require_cuda(x, gy)
    B, Hi, Wi, Ci = x.shape
    _, Ho, Wo, Co = gy.shape
    shape = (k * k, Ci, Co) if transposed else (k * k, Co, Ci)
    gw = torch.empty(shape, dtype=torch.float32, device=x.device)
    impl = 1 if CONV_IMPL == 1 else (3 if CONV_IMPL == 3 else WGRAD_IMPL)
    path = lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl)
    xin, gin = _tc_operand(x, path, x_planes), _tc_operand(gy, path)
    if impl == 3 and path != 3:
        impl = 1                               # shape outside the tensor-core path: exact fp32 SIMT
    nws = lib.gifb200_conv2d_wgrad_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, impl)
    ws = _workspace(nws, x.device)
    _profiled(True, lambda: check(lib.gifb200_conv2d_wgrad(ptr(xin), ptr(gin), ptr(gw), B, Hi, Wi, Ci, Ho, Wo, Co, k, mode,
                                                          int(flip), int(transposed), impl, ptr(ws), nws, stream()),
                                  "gifb200_conv2d_wgrad"),
              "wgrad", ("wgrad", mode, B, Hi, Wi, Ci, Co, k), (Ho, Wo))
    return gw


def _x3_backward_on_planes(x_shape, gy_shape, k, mode):
    """True when, in bf16x3 mode, BOTH consumers of a convolution's output gradient -- the input-gradient convolution and the
    weight gradient -- run on the tensor cores for these shapes, i.e. read only the split planes of gy (never its fp32 form)."""
    if CONV_IMPL != 3:
        return False
    B, Hi, Wi, Ci = x_shape
    _, Ho, Wo, Co = gy_shape
    if lib.gifb200_conv2d_workspace_bytes(B, Ho, Wo, Co, Hi, Wi, Ci, k, _ADJ_MODE[mode], 1, 3) == 0:
        return False
    return lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, 3) == 3


class _Conv(torch.autograd.Function):
    """y = conv(x; W) with W addressed in the physical buffer w[T][R][S] (see gifb200.h).  With ``act`` = (slope, gain, rt),
    y = lrelu(conv(x; w) + bias, slope) * gain in ONE kernel (fused epilogue of gifb200_conv2d; ``bias`` may be None):
    ConvLayer = EqualConv2d -> FusedLeakyReLU (cl.py:752-799), nn.Conv2d(+ReLU) of NoiseInjection (cl.py:405-414).  The
    backward is composed of the differentiable primitives (activation backward from the saved OUTPUT, adjoint conv, wgrad)."""

    @staticmethod
    def forward(ctx, x_arg, w, bias, k, mode, flip, transposed, out_hw, act):
        x, w = _c(x_arg), _c(w)
        epilogue = None if act is None else (None if bias is None else _c(bias.reshape(-1)),) + act
        y, x_used = _conv_raw(x, w, k, mode, flip, transposed, out_hw, epilogue)
        # the (possibly tf32-rounded) operand is what wgrad re-reads; a rounded copy is outside the autograd graph, so a
        # recorded (create_graph) backward takes the weight gradient of the input itself (_wgrad_raw rounds it again)
        ctx.save_for_backward(x_used, w, x_arg if x_used is not x and ctx.needs_input_grad[0] else None,
                              None if act is None else y)
        ctx.cfg = (k, mode, flip, transposed, tuple(x.shape[1:3]), _is_tf32(x_used), act,
                   None if bias is None else bias.shape)
        c = getattr(x_used, "_gifb200_planes", None)
        ctx.planes = c[1] if c is not None and c[0] == x_used._version else None   # bf16x3: wgrad reuses the split
        ctx.wprep = getattr(w, "_gifb200_prep", None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w, x_arg, y = ctx.saved_tensors
        k, mode, flip, transposed, in_hw, x_tf32, act, bias_shape = ctx.cfg
        _tag(x, x_tf32)
        _carry_planes(x, ctx.planes)
        if ctx.wprep is not None:
            w._gifb200_prep = ctx.wprep              # the input-gradient convolution reuses the staged-weight cache
        gx = gw = gb = None
        if act is not None:                          # gy becomes the gradient w.r.t. the pre-activation
            slope, gain, _ = act
            want_b = bias_shape is not None and ctx.needs_input_grad[2]
            if not torch.is_grad_enabled():
                # first-order backward: activation backward and bias gradient in one pass over (gy, y); in bf16x3 mode
                # the pass writes the dgrad / wgrad operand (split planes) directly, no fp32 copy
                gy = _c(gy)
                C = gy.shape[-1]
                carrier = C % 32 == 0 and _x3_backward_on_planes(x.shape, gy.shape, k, mode)
                gy, _, gb, _ = _tail_bwd(gy, y, y, None, 1, gy.numel() // max(C, 1), C, slope, gain,
                                         gt="planes" if carrier else "fp32", gb=want_b)
            else:
                gy = act_bwd(gy, y, slope, gain, rt=tf32_enabled())
                if want_b and _WEIGHT_GRADS[0]:
                    gb = rows_sum(gy.reshape(1, -1, gy.shape[-1]))
            gb = None if gb is None else gb.reshape(bias_shape)
        if ctx.needs_input_grad[0]:
            # adj(S1, f, t) = (S1, !f, !t); adj(S2, f, t) = (T2, f, !t); adj(T2, f, t) = (S2, f, !t)
            gx = _Conv.apply(gy, w, None, k, _ADJ_MODE[mode], (not flip) if mode == S1 else flip, not transposed, in_hw,
                             None)
        if ctx.needs_input_grad[1] and _WEIGHT_GRADS[0]:
            xw = x_arg if x_arg is not None and torch.is_grad_enabled() else x
            gw = _ConvWgrad.apply(xw, gy, k, mode, flip, transposed)
        return gx, gw, gb, None, None, None, None, None, None


class _ConvWgrad(torch.autograd.Function):
    """gw (physical layout of w) = d<gy, conv(x; w)>/dw -- bilinear in (x, gy)."""

    @staticmethod
    def forward(ctx, x, gy, k, mode, flip, transposed):
        x, gy = _c(x), _c(gy)
        ctx.save_for_backward(x, gy)
        ctx.cfg = (k, mode, flip, transposed)
        return _wgrad_raw(x, gy, k, mode, flip, transposed)

    @staticmethod
    def backward(ctx, ggw):
        x, gy = ctx.saved_tensors
        k, mode, flip, transposed = ctx.cfg
        gx = ggy = None
        if ctx.needs_input_grad[0]:   # <ggw, wgrad(x, gy)> = <gy, conv(x; ggw)>  ->  d/dx = adj conv of gy with ggw
            gx = _Conv.apply(gy, ggw, None, k, _ADJ_MODE[mode], (not flip) if mode == S1 else flip, not transposed,
                             tuple(x.shape[1:3]), None)
        if ctx.needs_input_grad[1]:
            ggy = _Conv.apply(x, ggw, None, k, mode, flip, transposed, tuple(gy.shape[1:3]), None)
        return gx, ggy, None, None, None, None


def conv2d_bias_act(x, w, bias, k, mode=S1, slope=0.2, gain=math.sqrt(2.0), rt=False):
    """Fused conv + bias + leaky-ReLU*gain (slope=1, gain=1: plain bias add; slope=0: ReLU)."""
    hi, wi = x.shape[1:3]
    out_hw = (conv_out_size(hi, k, mode), conv_out_size(wi, k, mode))
    return _tag(_Conv.apply(x, w, bias, k, mode, False, False, out_hw, (float(slope), float(gain), bool(rt))), rt)


def conv2d(x, w, k, mode=S1, flip=False, transposed=False):
    """x (B,H,W,Ci) NHWC, w (k*k, Co, Ci) tap-major [or (k*k, Ci, Co) with transposed=True] -> (B,Ho,Wo,Co)."""
    hi, wi = x.shape[1:3]
    return _Conv.apply(x, w, None, k, mode, flip, transposed, (conv_out_size(hi, k, mode), conv_out_size(wi, k, mode)),
                       None)


_NO_WEIGHT_CACHE = False    # tests set this to compare against prepare-and-stage on every call (as cache=False)
_prep_cache = {}     # (id of the parameter, view offset, shape, scale) -> (weakref to the parameter, its version, buffer, serial,
                     #                                                  address of the weight)
_stage_cache = {}    # (prep key, flip, transposed, impl, conv shape) -> [prep serial it was staged from, persistent workspace]
_prep_serial = [0]   # bumped on every recomputation: what the staged-operand cache compares (immune to address / id reuse)


class _PrepWeight(torch.autograd.Function):
    """(Co,Ci,k,k) parameter -> tap-major (k*k, Co, Ci) * scale, computed ONCE per parameter version: a network's weights
    change once per optimiser step but every layer is evaluated 3-5 times per step (D: three forwards), so the permute +
    scale (and, downstream, the staging of the tensor-core B operand, ``_stage_cache``) are shared by those calls.
    The result lives in ONE persistent buffer per parameter, rewritten in place when the parameter's version changes: a
    captured CUDA graph therefore always reads the buffer the (captured) recomputation of the current step wrote, whatever
    the hit / miss pattern was at capture time.  An autograd graph that still holds the old contents when the buffer is
    rewritten fails loudly (torch's version check), it cannot silently read new weights."""

    @staticmethod
    def forward(ctx, weight, scale):
        co, ci, kh, kw = weight.shape
        ctx.cfg = (co, ci, kh, kw, scale)
        base = weight._base if weight._base is not None else weight          # ``self.weight[0]`` is a view of the parameter
        key = (id(base), weight.storage_offset(), (co, ci, kh, kw), float(scale))
        hit = _prep_cache.get(key)
        # identity is checked through a weak reference: ids and addresses are reused once a network is freed, and a new
        # parameter that lands on an old one's id with an equal version counter must not see its prepared weights.
        # ``p.data = t`` rebinds the parameter to other storage without bumping its version: the address tells.
        if hit is None or hit[0]() is not base or hit[1] != weight._version or hit[4] != weight.data_ptr():
            same = hit is not None and hit[0]() is base
            buf = hit[2] if same else torch.empty((kh * kw, co, ci), dtype=torch.float32, device=weight.device)
            torch.mul(weight.detach().permute(2, 3, 0, 1), scale, out=buf.view(kh, kw, co, ci))    # one kernel, in place
            _prep_serial[0] += 1
            hit = (weakref.ref(base), weight._version, buf, _prep_serial[0], weight.data_ptr())
            _prep_cache[key] = hit
            if len(_prep_cache) > 4096:                                        # entries of freed networks
                for k_ in [k_ for k_, v_ in _prep_cache.items() if v_[0]() is None]:
                    del _prep_cache[k_]
                    for sk in [sk for sk in _stage_cache if sk[0] == k_]:
                        del _stage_cache[sk]
        alias = hit[2].detach()                 # a new tensor object on the cached storage: each call gets its own grad_fn
        alias._gifb200_prep = (key, hit[3])
        return alias

    @staticmethod
    def backward(ctx, g):
        co, ci, kh, kw, scale = ctx.cfg
        return (g.reshape(kh, kw, co, ci) * scale).permute(2, 3, 0, 1), None


def prep_weight(weight, scale=1.0, cache=True):
    """(Co,Ci,k,k) parameter -> tap-major (k*k, Co, Ci) * scale (differentiable; cached per parameter version).
    cache=False (the layers pass ``self.training``): prepare and stage on every call.  An eval-mode copy such as the EMA
    generator is updated by code that writes through ``.data`` (the reference's ``accumulate``), which no version counter
    sees."""
    if cache and weight.is_cuda and weight.dtype == torch.float32 and not _NO_WEIGHT_CACHE:
        return _PrepWeight.apply(weight, float(scale))
    co, ci, kh, kw = weight.shape
    return (weight * scale).permute(2, 3, 0, 1).reshape(kh * kw, co, ci).contiguous()


def _staged_workspace(w, nws, flip, transposed, impl, shape_key, device):
    """The persistent workspace holding the staged B operand of a cached prepared weight, and whether it is current
    (GIFB200_CONV_PRESTAGED).  Weights that do not come out of ``prep_weight``'s cache use the shared scratch workspace."""
    tag = getattr(w, "_gifb200_prep", None)
    if tag is None or nws == 0:
        return _workspace(nws, device), False
    pkey, serial = tag
    key = (pkey, bool(flip), bool(transposed), impl, shape_key)
    ent = _stage_cache.get(key)
    if ent is None or ent[1].numel() < nws:
        if ent is not None:
            _ws_retired.append(ent[1])           # retired, never freed: a captured CUDA graph may hold its address
        ent = [None, torch.empty(nws, dtype=torch.uint8, device=device)]
        _stage_cache[key] = ent
    fresh = ent[0] == serial
    ent[0] = serial
    return ent[1], fresh


# --------------------------------------------------------------------------------------------- upfirdn2d
def upfirdn_out_size(h, kh, up, down, p0, p1):
    return (h * up + p0 + p1 - kh) // down + 1


class _UpFirDn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, kernel, up, down, py0, px0, out_hw, flip, rt):
        x = _c(x)
        require_cuda(x, kernel)
        B, Hi, Wi, C = x.shape
        kh, kw = kernel.shape
        Ho, Wo = out_hw
        y = torch.empty((B, Ho, Wo, C), dtype=torch.float32, device=x.device)
        check(lib.gifb200_upfirdn2d(ptr(x), ptr(kernel), ptr(y), B, Hi, Wi, C, Ho, Wo, kh, kw, up, down, py0, px0,
                                    int(flip), int(rt), stream()), "gifb200_upfirdn2d")
        ctx.kernel = kernel
        ctx.cfg = (up, down, py0, px0, (Hi, Wi), flip, kh, kw)
        return y

    @staticmethod
    def backward(ctx, gy):
        up, down, py0, px0, in_hw, flip, kh, kw = ctx.cfg
        # adjoint: swap up/down, reverse the kernel, pad0' = k-1-pad0, output size = forward's input size (SURVEY A1)
        rt = tf32_enabled()
        gx = _tag(_UpFirDn.apply(gy, ctx.kernel, down, up, kh - 1 - py0, kw - 1 - px0, in_hw, not flip, rt), rt)
        return gx, None, None, None, None, None, None, None, None


def upfirdn2d(x, kernel, up=1, down=1, pad=(0, 0), rt=False):
    """NHWC equivalent of cl.py:42-72 (same pad on both axes, cl.py:53).  rt: round the output to tf32."""
    kernel = _c(kernel.detach().to(torch.float32))
    kh, kw = kernel.shape
    ho = upfirdn_out_size(x.shape[1], kh, up, down, pad[0], pad[1])
    wo = upfirdn_out_size(x.shape[2], kw, up, down, pad[0], pad[1])
    return _tag(_UpFirDn.apply(x, kernel, up, down, pad[0], pad[0], (ho, wo), False, rt), rt)


# --------------------------------------------------------------------------------------------- bias / act
def _grad_planes(C, P):
    """True when an elementwise gradient of C channels and P pixels per image goes on to bf16x3 tensor-core contractions:
    its producer then writes the split planes in the same pass, which saves the split pass's read."""
    return CONV_IMPL == 3 and C % 32 == 0 and P >= 256


def _tail_bwd(gy, y, acc, d, B, P, C, slope, gain, gt=None, gacc=None, gb=False, gd=False):
    """The fused first-order tail backward (gifb200_tail_bwd, or gifb200_tail_bwd_planes when any planes are wanted) on
    contiguous tensors.  gt, gacc: None (not computed), "fp32", "both" (fp32 and planes) or "planes" (an unwritten fp32
    tensor carrying the planes: only for the two tensor-core contractions of _x3_backward_on_planes); gb, gd: whether the
    bias / modulation gradient is computed.  Returns (gt, gacc, gb (C,), gd (B, C)), None for what was not computed."""
    outs = [None if m is None else torch.empty_like(gy) for m in (gt, gacc)]
    gbt = torch.empty(C, dtype=torch.float32, device=gy.device) if gb else None
    gdt = torch.empty((B, C), dtype=torch.float32, device=gy.device) if gd else None
    fp32 = [t if m in ("fp32", "both") else None for t, m in zip(outs, (gt, gacc))]
    planes = [torch.empty((2,) + tuple(gy.shape), dtype=torch.bfloat16, device=gy.device) if m in ("planes", "both")
              else None for m in (gt, gacc)]
    if planes[0] is not None or planes[1] is not None:
        rt = False                                   # the planes entry point does not round its fp32 outputs
        check(lib.gifb200_tail_bwd_planes(ptr(gy), ptr(y), ptr(acc), ptr(d), ptr(fp32[0]), ptr(fp32[1]), ptr(gbt), ptr(gdt),
                                          B, P, C, slope, gain, ptr(planes[0]), ptr(planes[1]), stream()),
              "gifb200_tail_bwd_planes")
    else:
        rt = tf32_enabled()
        check(lib.gifb200_tail_bwd(ptr(gy), ptr(y), ptr(acc), ptr(d), ptr(fp32[0]), ptr(fp32[1]), ptr(gbt), ptr(gdt), B, P, C,
                                   slope, gain, int(rt), stream()), "gifb200_tail_bwd")
    for t, pl in zip(outs, planes):
        if t is not None:
            _carry_planes(t, pl)
            _tag(t, rt)
    return outs[0], outs[1], gbt, gdt


def _scale_bwd(gy, x, s, rt=False):
    """The fused first-order backward of y = x*s[b,c] (gifb200_scale_bwd) on contiguous tensors: (gx = gy*s, gs = sum_p gy*x);
    rt: round gx to tf32."""
    B, C = gy.shape[0], gy.shape[-1]
    P = gy.numel() // max(B * C, 1)
    gx = torch.empty_like(gy)
    gs = torch.empty((B, C), dtype=torch.float32, device=gy.device)
    check(lib.gifb200_scale_bwd(ptr(gy), ptr(x), ptr(s), ptr(gx), ptr(gs), B, P, C, int(rt), stream()), "gifb200_scale_bwd")
    return _tag(gx, rt), gs


class _BiasAct(torch.autograd.Function):
    """y = lrelu(x*rowscale[b,c] + add + bias[c], slope) * gain  (rowscale/add/bias optional)."""

    @staticmethod
    def forward(ctx, x, rowscale, add, bias, slope, gain, rt):
        x = _c(x)
        rowscale = None if rowscale is None else _c(rowscale)
        add = None if add is None else _c(add)
        bias_flat = None if bias is None else _c(bias.reshape(-1))
        require_cuda(x, rowscale, add, bias_flat)
        B, C = x.shape[0], x.shape[-1]
        P = x.numel() // max(B * C, 1)
        y = torch.empty_like(x)
        check(lib.gifb200_bias_act(ptr(x), ptr(rowscale), ptr(add), ptr(bias_flat), ptr(y), B, P, C, slope, gain,
                                   int(rt), stream()), "gifb200_bias_act")
        ctx.save_for_backward(x, rowscale, y)
        ctx.cfg = (slope, gain, None if bias is None else bias.shape, add is not None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, rowscale, y = ctx.saved_tensors
        slope, gain, bias_shape, has_add = ctx.cfg
        if not torch.is_grad_enabled():
            # first-order backward only (no create_graph): one fused pass instead of act_bwd + chan_scale + spatial_dot + rows_sum
            gy = _c(gy)
            B, C = gy.shape[0], gy.shape[-1]
            P = gy.numel() // max(B * C, 1)
            want_b = bias_shape is not None and ctx.needs_input_grad[3]
            # bf16x3: the gradients leave on autograd edges towards convolutions (the modulated conv and the noise branch)
            # or FIR filters: write the fp32 form AND the split planes in the same pass
            x3 = _grad_planes(C, P)
            gt, gacc, gb, gd = _tail_bwd(gy, y, x, rowscale, B, P, C, slope, gain, gt="both" if x3 and has_add else "fp32",
                                         gacc=None if rowscale is None else ("both" if x3 else "fp32"), gb=want_b,
                                         gd=rowscale is not None and ctx.needs_input_grad[1])
            gx = (gacc if rowscale is not None else gt) if ctx.needs_input_grad[0] else None
            return (gx, gd, gt if (has_add and ctx.needs_input_grad[2]) else None,
                    gb.reshape(bias_shape) if want_b else None, None, None, None)
        if not _WEIGHT_GRADS[0] and rowscale is not None:
            # input_gradient_only (path-length pass): one node, fused second-order rule; no noise-branch / bias gradients
            gx, grs = _TailBwdCG.apply(gy, y, x, rowscale, slope, gain, True)
            return (gx if ctx.needs_input_grad[0] else None, grs if ctx.needs_input_grad[1] else None, None, None, None, None,
                    None)
        gt = act_bwd(gy, y, slope, gain, rt=tf32_enabled())   # gradient w.r.t. the pre-activation t (feeds dgrad/wgrad)
        gx = grs = gadd = gb = None
        if ctx.needs_input_grad[0]:
            gx = gt if rowscale is None else chan_scale(gt, rowscale)
        if rowscale is not None and ctx.needs_input_grad[1]:
            grs = spatial_dot(gt, x)
        if has_add and ctx.needs_input_grad[2]:
            gadd = gt
        if bias_shape is not None and ctx.needs_input_grad[3] and _WEIGHT_GRADS[0]:
            gb = rows_sum(gt.reshape(1, -1, gt.shape[-1])).reshape(bias_shape)
        return gx, grs, gadd, gb, None, None, None


class _TailBwdCG(torch.autograd.Function):
    """The first-order backward of the StyledConv tail (y given: gacc = gy*m(y)*d, gd = sum_p gy*m(y)*acc) or of the input
    modulation (y None: m = 1) as ONE differentiable node with a fused second-order pass (gifb200_tail_bwd2), for the
    create_graph pass of the path-length regulariser -- instead of act_bwd + chan_scale + spatial_dot, whose recorded graph
    costs five more elementwise kernels and autograd's gradient-sum adds per layer in the double backward.  Only taken inside
    ``input_gradient_only()`` (the noise-branch and bias gradients are not produced).  Second order is the last: its
    backward is not differentiable again."""

    @staticmethod
    def forward(ctx, gy, y, acc, d, slope, gain, want_planes):
        gy, acc, d = _c(gy), _c(acc), _c(d)
        require_cuda(gy, acc, d)
        if y is None:
            gacc, gd = _scale_bwd(gy, acc, d)
        else:
            y = _c(y)
            B, C = gy.shape[0], gy.shape[-1]
            P = gy.numel() // max(B * C, 1)
            _, gacc, _, gd = _tail_bwd(gy, y, acc, d, B, P, C, slope, gain,
                                       gacc="both" if want_planes and _grad_planes(C, P) else "fp32", gd=True)
        ctx.save_for_backward(gy, y, acc, d)
        ctx.cfg = (slope, gain, y is not None)
        ctx.set_materialize_grads(False)
        return gacc, gd

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gg, ggd):
        gy, y, acc, d = ctx.saved_tensors
        slope, gain, has_y = ctx.cfg
        if gg is None and ggd is None:
            return None, None, None, None, None, None, None
        gg = None if gg is None else _c(gg)
        ggd = None if ggd is None else _c(ggd)
        B, C = gy.shape[0], gy.shape[-1]
        P = gy.numel() // max(B * C, 1)
        ggy = torch.empty_like(gy) if ctx.needs_input_grad[0] else None
        gx2 = torch.empty_like(gy) if (ctx.needs_input_grad[2] and ggd is not None) else None
        gdd = torch.empty((B, C), dtype=torch.float32, device=gy.device) if (ctx.needs_input_grad[3] and gg is not None) else None
        pp = None
        if ggy is not None and not has_y and _grad_planes(C, P):
            pp = torch.empty((2,) + tuple(gy.shape), dtype=torch.bfloat16, device=gy.device)   # gy came out of a convolution
        check(lib.gifb200_tail_bwd2(ptr(gg), ptr(ggd), ptr(gy), ptr(y) if has_y else None, ptr(acc), ptr(d), ptr(ggy), ptr(gx2),
                                    ptr(gdd), B, P, C, slope, gain, ptr(pp), stream()), "gifb200_tail_bwd2")
        _carry_planes(ggy, pp)
        return ggy, None, gx2, gdd, None, None, None


class _ActBwd(torch.autograd.Function):
    """gx = gy * gain * (y > 0 ? 1 : slope): linear in gy, piecewise constant in y."""

    @staticmethod
    def forward(ctx, gy, y, slope, gain, rt):
        gy = _c(gy)
        require_cuda(gy, y)
        gx = torch.empty_like(gy)
        check(lib.gifb200_act_bwd(ptr(gy), ptr(y), ptr(gx), gy.numel(), slope, gain, int(rt), stream()),
              "gifb200_act_bwd")
        ctx.save_for_backward(y)
        ctx.cfg = (slope, gain, rt)
        return gx

    @staticmethod
    def backward(ctx, ggx):
        (y,) = ctx.saved_tensors
        slope, gain, rt = ctx.cfg
        return _tag(_ActBwd.apply(ggx, y, slope, gain, rt), rt), None, None, None, None


def act_bwd(gy, y, slope, gain, rt=False):
    return _tag(_ActBwd.apply(gy, y, slope, gain, rt), rt)


def bias_act(x, bias=None, slope=0.2, gain=math.sqrt(2.0), rowscale=None, add=None, rt=False):
    """rt: round the output to tf32 (set when the consumer is a tensor-core convolution)."""
    return _tag(_BiasAct.apply(x, rowscale, add, bias, float(slope), float(gain), rt), rt)


class _RowsSum(torch.autograd.Function):
    """(G, rows, C) -> (G, C)."""

    @staticmethod
    def forward(ctx, x):
        x = _c(x)
        require_cuda(x)
        G, rows, C = x.shape
        out = torch.empty((G, C), dtype=torch.float32, device=x.device)
        check(lib.gifb200_rows_sum(ptr(x), ptr(out), G, rows, C, stream()), "gifb200_rows_sum")
        ctx.shape = x.shape
        return out

    @staticmethod
    def backward(ctx, g):
        return g[:, None, :].expand(ctx.shape)


def rows_sum(x):
    return _RowsSum.apply(x)


# --------------------------------------------------------------------------------------------- modulation
class _ChanScale(torch.autograd.Function):
    """y[b,...,c] = x[b,...,c] * s[b,c]."""

    @staticmethod
    def forward(ctx, x, s, round_tf32):
        x, s = _c(x), _c(s)
        require_cuda(x, s)
        B, C = x.shape[0], x.shape[-1]
        P = x.numel() // max(B * C, 1)
        y = torch.empty_like(x)
        check(lib.gifb200_chan_scale(ptr(x), ptr(s), ptr(y), B, P, C, int(round_tf32), stream()), "gifb200_chan_scale")
        ctx.save_for_backward(x, s)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, s = ctx.saved_tensors
        if not torch.is_grad_enabled() and ctx.needs_input_grad[0] and ctx.needs_input_grad[1]:
            gx, gs = _scale_bwd(_c(gy), x, s, tf32_enabled())     # fused first-order pass: gx = gy*s, gs = sum gy*x
            return gx, gs, None
        if torch.is_grad_enabled() and not _WEIGHT_GRADS[0] and ctx.needs_input_grad[0] and ctx.needs_input_grad[1]:
            gx, gs = _TailBwdCG.apply(gy, None, x, s, 1.0, 1.0, False)     # one node, fused second-order rule
            return gx, gs, None
        gx = chan_scale(gy, s, tf32_enabled()) if ctx.needs_input_grad[0] else None
        gs = spatial_dot(gy, x) if ctx.needs_input_grad[1] else None
        return gx, gs, None


class _SpatialDot(torch.autograd.Function):
    """out[b,c] = sum_pixels a*b."""

    @staticmethod
    def forward(ctx, a, b):
        a, b = _c(a), _c(b)
        require_cuda(a, b)
        B, C = a.shape[0], a.shape[-1]
        P = a.numel() // max(B * C, 1)
        out = torch.empty((B, C), dtype=torch.float32, device=a.device)
        check(lib.gifb200_spatial_dot(ptr(a), ptr(b), ptr(out), B, P, C, stream()), "gifb200_spatial_dot")
        ctx.save_for_backward(a, b)
        return out

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        ga = chan_scale(b, g) if ctx.needs_input_grad[0] else None
        gb = chan_scale(a, g) if ctx.needs_input_grad[1] else None
        return ga, gb


def chan_scale(x, s, round_tf32=False):
    return _tag(_ChanScale.apply(x, s, round_tf32), round_tf32)


class _ModConvX3(torch.autograd.Function):
    """y = conv(x * s[b, :]; w) in the bf16x3 mode with the modulation fused into the operand split: ONE pass reads x and
    writes the two bf16 planes of x*s (gifb200_split_bf16 with a scale vector), the tensor-core kernel reads those; the
    fp32 modulated copy of the input (2 x 1.07 GB per 256^2 layer) never exists.  First-order backward: input-gradient
    convolution + the fused scale_bwd pass + weight gradient on the saved planes; when a higher derivative is being recorded
    (path-length regulariser) the backward is the closed set of differentiable ops (chan_scale, conv, wgrad, spatial_dot)."""

    @staticmethod
    def forward(ctx, x, s, w, k, mode, out_hw):
        x, s, w = _c(x), _c(s), _c(w)
        require_cuda(x, s, w)
        B, C = x.shape[0], x.shape[-1]
        P = x.numel() // max(B * C, 1)
        pl = torch.empty((2,) + tuple(x.shape), dtype=torch.bfloat16, device=x.device)
        check(lib.gifb200_split_bf16(ptr(x), ptr(s), ptr(pl), B, P, C, stream()), "gifb200_split_bf16(scale)")
        y, _ = _conv_raw(x, w, k, mode, False, False, out_hw, planes=pl)
        ctx.save_for_backward(x, s, w)
        ctx.planes = pl
        ctx.wprep = getattr(w, "_gifb200_prep", None)
        ctx.cfg = (k, mode, tuple(x.shape[1:3]))
        return y

    @staticmethod
    def backward(ctx, gy):
        x, s, w = ctx.saved_tensors
        k, mode, in_hw = ctx.cfg
        if ctx.wprep is not None:
            w._gifb200_prep = ctx.wprep
        adj = (gy, w, None, k, _ADJ_MODE[mode], mode == S1, True, in_hw, None)
        if torch.is_grad_enabled():
            gxs = _Conv.apply(*adj) if (ctx.needs_input_grad[0] or ctx.needs_input_grad[1]) else None
            if not _WEIGHT_GRADS[0] and gxs is not None:
                gx, gs = _TailBwdCG.apply(gxs, None, x, s, 1.0, 1.0, False)
                return gx, gs, None, None, None, None
            gx = chan_scale(gxs, s) if ctx.needs_input_grad[0] else None
            gs = spatial_dot(gxs, x) if ctx.needs_input_grad[1] else None
            gw = None
            if ctx.needs_input_grad[2] and _WEIGHT_GRADS[0]:
                gw = _ConvWgrad.apply(chan_scale(x, s), gy, k, mode, False, False)
            return gx, gs, gw, None, None, None
        gy = _c(gy)
        gx = gs = gw = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            gxs, _ = _conv_raw(gy, w, k, _ADJ_MODE[mode], mode == S1, True, in_hw)
            gx, gs = _scale_bwd(gxs, x, s)
        if ctx.needs_input_grad[2] and _WEIGHT_GRADS[0]:
            gw = _wgrad_raw(x, gy, k, mode, False, False, x_planes=ctx.planes)
        return gx, gs, gw, None, None, None


def modconv(x, s, w, k, mode):
    """conv(x * s; w): the modulate-input form of ModulatedConv2d (cl.py:311-347).  bf16x3 + a tensor-core shape: the fused
    split (no modulated fp32 copy); otherwise chan_scale followed by conv2d."""
    hi, wi = x.shape[1:3]
    out_hw = (conv_out_size(hi, k, mode), conv_out_size(wi, k, mode))
    if CONV_IMPL == 3 and x.shape[-1] % 4 == 0:
        B, Ci = x.shape[0], x.shape[-1]
        Co = w.shape[1]
        if lib.gifb200_conv2d_workspace_bytes(B, hi, wi, Ci, out_hw[0], out_hw[1], Co, k, mode, 0, 3) > 0 and \
                lib.gifb200_conv2d_wgrad_path(B, hi, wi, Ci, out_hw[0], out_hw[1], Co, k, mode, 3) == 3:
            return _ModConvX3.apply(x, s, w, k, mode, out_hw)
    return conv2d(chan_scale(x, s, tf32_enabled()), w, k, mode)


def spatial_dot(a, b):
    return _SpatialDot.apply(a, b)


class _Axpby(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b, alpha, beta, rt):
        a = _c(a)
        b = None if b is None else _c(b)
        require_cuda(a, b)
        y = torch.empty_like(a)
        check(lib.gifb200_axpby(ptr(a), ptr(b), ptr(y), a.numel(), alpha, beta, int(rt), stream()), "gifb200_axpby")
        ctx.cfg = (alpha, beta, b is not None)
        return y

    @staticmethod
    def backward(ctx, g):
        alpha, beta, has_b = ctx.cfg
        rt = tf32_enabled()
        ga = _tag(_Axpby.apply(g, None, alpha, 0.0, rt), rt) if ctx.needs_input_grad[0] else None
        if has_b and ctx.needs_input_grad[1]:
            # the residual merge (a + b)/sqrt2 has alpha == beta: both branches receive the same tensor, computed once
            gb = ga if (ga is not None and alpha == beta) else _tag(_Axpby.apply(g, None, beta, 0.0, rt), rt)
        else:
            gb = None
        return ga, gb, None, None, None


def axpby(a, b, alpha=1.0, beta=1.0, rt=False):
    """alpha*a + beta*b on same-shape tensors."""
    return _tag(_Axpby.apply(a, b, float(alpha), float(beta), rt), rt)


class _Demod(torch.autograd.Function):
    """d[b,o] = rsqrt(sum_i s[b,i]^2 q[o,i] + eps)  (cl.py:315-316).  Forward: warp-shuffle kernel; the O(B*Ci*Co)
    backward is expressed with differentiable torch ops on these tiny matrices."""

    @staticmethod
    def forward(ctx, s, q, eps):
        s, q = _c(s), _c(q)
        require_cuda(s, q)
        B, Ci = s.shape
        Co = q.shape[0]
        d = torch.empty((B, Co), dtype=torch.float32, device=s.device)
        check(lib.gifb200_demod(ptr(s), ptr(q), ptr(d), B, Ci, Co, eps, stream()), "gifb200_demod")
        ctx.save_for_backward(s, q, d)
        return d

    @staticmethod
    def backward(ctx, gd):
        s, q, d = ctx.saved_tensors
        t = -0.5 * gd * d * d * d                          # d(d)/d(sum) = -1/2 d^3
        gs = 2.0 * s * matmul(t, q) if ctx.needs_input_grad[0] else None
        gq = matmul(t, s * s, trans_a=True) if ctx.needs_input_grad[1] else None
        return gs, gq, None


def demod(s, q, eps=1e-8):
    return _Demod.apply(s, q, float(eps))


# --------------------------------------------------------------------------------------------- ToRGB
class _ToRgbFwd(torch.autograd.Function):
    """y[b,p,k] = sum_i x[b,p,i] ws[b,k,i]  (k = 0..2)."""

    @staticmethod
    def forward(ctx, x, ws):
        x, ws = _c(x), _c(ws)
        require_cuda(x, ws)
        B, C = x.shape[0], x.shape[-1]
        P = x.numel() // max(B * C, 1)
        y = torch.empty(x.shape[:-1] + (3,), dtype=torch.float32, device=x.device)
        check(lib.gifb200_torgb_fwd(ptr(x), ptr(ws), ptr(y), B, P, C, stream()), "gifb200_torgb_fwd")
        ctx.save_for_backward(x, ws)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, ws = ctx.saved_tensors
        gx = _ToRgbBwdX.apply(gy, ws) if ctx.needs_input_grad[0] else None
        gws = _ToRgbBwdW.apply(gy, x) if ctx.needs_input_grad[1] else None
        return gx, gws


class _ToRgbBwdX(torch.autograd.Function):
    """gx[b,p,i] = sum_k gy[b,p,k] ws[b,k,i]."""

    @staticmethod
    def forward(ctx, gy, ws):
        gy, ws = _c(gy), _c(ws)
        require_cuda(gy, ws)
        B, C = ws.shape[0], ws.shape[-1]
        P = gy.numel() // max(B * 3, 1)
        gx = torch.empty(gy.shape[:-1] + (C,), dtype=torch.float32, device=gy.device)
        check(lib.gifb200_torgb_bwd_x(ptr(gy), ptr(ws), ptr(gx), B, P, C, stream()), "gifb200_torgb_bwd_x")
        ctx.save_for_backward(gy, ws)
        return gx

    @staticmethod
    def backward(ctx, g):
        gy, ws = ctx.saved_tensors
        ggy = _ToRgbFwd.apply(g, ws) if ctx.needs_input_grad[0] else None
        gws = _ToRgbBwdW.apply(gy, g) if ctx.needs_input_grad[1] else None
        return ggy, gws


class _ToRgbBwdW(torch.autograd.Function):
    """gws[b,k,i] = sum_p gy[b,p,k] x[b,p,i]."""

    @staticmethod
    def forward(ctx, gy, x):
        gy, x = _c(gy), _c(x)
        require_cuda(gy, x)
        B, C = x.shape[0], x.shape[-1]
        P = x.numel() // max(B * C, 1)
        gws = torch.empty((B, 3, C), dtype=torch.float32, device=x.device)
        check(lib.gifb200_torgb_bwd_w(ptr(gy), ptr(x), ptr(gws), B, P, C, stream()), "gifb200_torgb_bwd_w")
        ctx.save_for_backward(gy, x)
        return gws

    @staticmethod
    def backward(ctx, g):
        gy, x = ctx.saved_tensors
        ggy = _ToRgbFwd.apply(x, g) if ctx.needs_input_grad[0] else None
        gx = _ToRgbBwdX.apply(gy, g) if ctx.needs_input_grad[1] else None
        return ggy, gx


def torgb(x, ws):
    return _ToRgbFwd.apply(x, ws)


# --------------------------------------------------------------------------------------------- small GEMM
def _sgemm_raw(a, b, trans_a, trans_b, alpha):
    a, b = _c(a), _c(b)
    require_cuda(a, b)
    M = a.shape[1] if trans_a else a.shape[0]
    K = a.shape[0] if trans_a else a.shape[1]
    N = b.shape[0] if trans_b else b.shape[1]
    assert (b.shape[1] if trans_b else b.shape[0]) == K, f"sgemm inner dims {tuple(a.shape)} x {tuple(b.shape)}"
    c = torch.empty((M, N), dtype=torch.float32, device=a.device)
    check(lib.gifb200_sgemm(int(trans_a), int(trans_b), M, N, K, alpha, ptr(a), a.shape[1], ptr(b), b.shape[1],
                            ptr(c), N, stream()), "gifb200_sgemm")
    return c


class _MatMul(torch.autograd.Function):
    """C = alpha * op(A) op(B)."""

    @staticmethod
    def forward(ctx, a, b, trans_a, trans_b, alpha):
        ctx.save_for_backward(a, b)
        ctx.cfg = (trans_a, trans_b, alpha)
        return _sgemm_raw(a, b, trans_a, trans_b, alpha)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        ta, tb, alpha = ctx.cfg
        ga = gb = None
        if ctx.needs_input_grad[0]:
            # C = op(A) op(B):  d/d op(A) = G op(B)^T ;  if A stored transposed: dA = (G op(B)^T)^T = op(B) G^T
            ga = _MatMul.apply(b, g, tb, True, alpha) if ta else _MatMul.apply(g, b, False, not tb, alpha)
        if ctx.needs_input_grad[1]:
            # d/d op(B) = op(A)^T G ; if B stored transposed: dB = G^T op(A)
            gb = _MatMul.apply(g, a, True, ta, alpha) if tb else _MatMul.apply(a, g, not ta, False, alpha)
        return ga, gb, None, None, None


def matmul(a, b, trans_a=False, trans_b=False, alpha=1.0):
    return _MatMul.apply(a, b, trans_a, trans_b, float(alpha))


# --------------------------------------------------------------------------------------------- cond pyramid
class _CondDown(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, s, adjoint, full_hw):
        x = _c(x)
        require_cuda(x)
        B, _, _, C = x.shape
        H, W = full_hw
        if not adjoint:
            y = torch.empty((B, H // s, W // s, C), dtype=torch.float32, device=x.device)
            check(lib.gifb200_cond_down(ptr(x), ptr(y), B, H, W, C, s, 0, stream()), "gifb200_cond_down")
        else:
            y = torch.empty((B, H, W, C), dtype=torch.float32, device=x.device)
            check(lib.gifb200_cond_down(ptr(y), ptr(x), B, H, W, C, s, 1, stream()), "gifb200_cond_down(adj)")
        ctx.cfg = (s, adjoint, full_hw)
        return y

    @staticmethod
    def backward(ctx, g):
        s, adjoint, full_hw = ctx.cfg
        return _CondDown.apply(g, s, not adjoint, full_hw), None, None, None


def cond_down(x, s):
    """(B,H,W,C) -> (B,H/s,W/s,C): bilinear (align_corners=False) reduction by a power of two (gen.py:309-314)."""
    if s == 1:
        return x
    return _CondDown.apply(x, s, False, tuple(x.shape[1:3]))


class _CondUp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, s, adjoint, small_hw):
        x = _c(x)
        require_cuda(x)
        B, _, _, C = x.shape
        H, W = small_hw
        if not adjoint:
            y = torch.empty((B, H * s, W * s, C), dtype=torch.float32, device=x.device)
            check(lib.gifb200_cond_up(ptr(x), ptr(y), B, H, W, C, s, 0, stream()), "gifb200_cond_up")
        else:
            y = torch.empty((B, H, W, C), dtype=torch.float32, device=x.device)
            check(lib.gifb200_cond_up(ptr(y), ptr(x), B, H, W, C, s, 1, stream()), "gifb200_cond_up(adj)")
        ctx.cfg = (s, adjoint, small_hw)
        return y

    @staticmethod
    def backward(ctx, g):
        s, adjoint, small_hw = ctx.cfg
        return _CondUp.apply(g, s, not adjoint, small_hw), None, None, None


def cond_up(x, s):
    """(B,H,W,C) -> (B,sH,sW,C): bilinear (align_corners=False) upsampling by a power of two, edges clamped as torch does."""
    if s == 1:
        return x
    return _CondUp.apply(x, s, False, tuple(x.shape[1:3]))


def cond_resize(x, size):
    """(B,H,W,C) -> (B,size,size,C) for a square power-of-two ratio: F.interpolate(x, (size, size), 'bilinear',
    align_corners=False) (gen.py:309-314).  Other ratios raise NotImplementedError."""
    full = x.shape[1]
    big, small = max(full, size), min(full, size)
    if x.shape[2] != full or big % small != 0 or (big // small) & (big // small - 1):
        raise NotImplementedError("gif_b200 condition pyramid: the condition and every level must differ by a power-of-two "
                                  f"factor (got {tuple(x.shape[1:3])} -> {size})")
    return cond_down(x, full // size) if full >= size else cond_up(x, size // full)


# --------------------------------------------------------------------------------------------- forward-only feature network ops
# The FID Inception network never needs gradients: these wrappers take no part in autograd and refuse inputs that require
# grad (under grad mode) instead of silently returning a result without a graph.
def _forward_only(what, *tensors):
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        raise RuntimeError(f"gif_b200.ops.{what} is forward-only: its inputs must not require grad")


def conv_ex_out_size(h, k, stride, pad):
    return (h + 2 * pad - k) // stride + 1


def conv2d_ex_impl(x_shape, co, kh, kw, stride, pad):
    """The gifb200_conv2d_ex impl the current precision mode runs for this shape: 1 (exact fp32), 2 (tf32) or 3 (bf16x3)."""
    if CONV_IMPL == 1:
        return 1
    B, Hi, Wi, Ci = x_shape
    Ho, Wo = conv_ex_out_size(Hi, kh, stride, pad[0]), conv_ex_out_size(Wi, kw, stride, pad[1])
    if lib.gifb200_conv2d_ex_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, co, kh, kw, stride, pad[0], pad[1], 2) == 0:
        return 1
    return 3 if CONV_IMPL == 3 else 2


def conv2d_ex(x, w, kh, kw, stride=1, pad=(0, 0), bias=None, relu=False, out=None, c0=0, round_tf32=False, workspace=None):
    """Forward-only general convolution (gifb200_conv2d_ex): x (B,H,W,Ci) channels-last, w (kh*kw, Co, Ci) tap-major,
    y = relu?(conv(x, w) + bias).  ``out`` (B,Ho,Wo,Cy): write channels [c0, c0+Co) of it instead of a new tensor.
    The precision mode (``set_precision``) picks the kernel; tensor-core inputs are rounded to tf32 or split into bf16
    planes (cached per tensor) here.  ``workspace``: a caller-kept ``[tensor or None, staged impl]`` list holding the staged
    weights of ``w`` between calls (GIFB200_CONV_PRESTAGED); None stages ``w`` on every call."""
    _forward_only("conv2d_ex", x, w, bias)
    require_cuda(x, w, bias)
    x = _c(x)
    B, Hi, Wi, Ci = x.shape
    T, Co, Ci_w = w.shape
    if T != kh * kw or Ci_w != Ci:
        raise ValueError(f"conv2d_ex: weight {tuple(w.shape)} vs kernel {kh}x{kw} and input channels {Ci}")
    if bias is not None and not relu:
        raise ValueError("conv2d_ex: the fused epilogue is bias + ReLU; a bias needs relu=True")
    Ho, Wo = conv_ex_out_size(Hi, kh, stride, pad[0]), conv_ex_out_size(Wi, kw, stride, pad[1])
    if out is None:
        out = torch.empty((B, Ho, Wo, Co), dtype=torch.float32, device=x.device)
    elif out.shape[:3] != (B, Ho, Wo) or not out.is_contiguous() or out.dtype != torch.float32:
        raise ValueError(f"conv2d_ex: out {tuple(out.shape)} is not a contiguous (B, {Ho}, {Wo}, Cy) float32 tensor")
    impl = conv2d_ex_impl(x.shape, Co, kh, kw, stride, pad)
    xin = _tc_operand(x, impl)
    nws = lib.gifb200_conv2d_ex_workspace_bytes(B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad[0], pad[1], impl)
    flag = 0
    if nws == 0:
        ws = None
    elif workspace is None:
        ws = _workspace(nws, x.device)
    else:
        if workspace[0] is None or workspace[0].numel() < nws or workspace[1] != impl:
            workspace[0], workspace[1] = torch.empty(nws, dtype=torch.uint8, device=x.device), impl
        else:
            flag = 0x10                                      # GIFB200_CONV_PRESTAGED: the staged weights are current
        ws = workspace[0]
    check(lib.gifb200_conv2d_ex(ptr(xin), ptr(_c(w)), ptr(out), B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad[0], pad[1],
                                out.shape[3], c0, impl | flag, int(relu), ptr(bias), int(round_tf32),
                                ptr(ws), nws, stream()), "gifb200_conv2d_ex")
    return out


def pool2d(x, op, stride, pad, out=None, c0=0, round_tf32=False):
    """Forward-only 3x3 pooling (gifb200_pool2d) of x (B,H,W,C): op "max" (padded cells -inf) or "avg"
    (count_include_pad=False); ``out``/``c0`` as in conv2d_ex."""
    _forward_only("pool2d", x)
    require_cuda(x)
    x = _c(x)
    B, Hi, Wi, C = x.shape
    Ho, Wo = conv_ex_out_size(Hi, 3, stride, pad), conv_ex_out_size(Wi, 3, stride, pad)
    if out is None:
        out = torch.empty((B, Ho, Wo, C), dtype=torch.float32, device=x.device)
    elif out.shape[:3] != (B, Ho, Wo) or not out.is_contiguous():
        raise ValueError(f"pool2d: out {tuple(out.shape)} is not a contiguous (B, {Ho}, {Wo}, Cy) tensor")
    check(lib.gifb200_pool2d(ptr(x), ptr(out), B, Hi, Wi, C, Ho, Wo, stride, pad, {"max": 0, "avg": 1}[op], out.shape[3], c0,
                             int(round_tf32), stream()), "gifb200_pool2d")
    return out


def resize_bilinear(x, size, channels=32, scale=1.0, shift=0.0, round_tf32=False):
    """Forward-only F.interpolate(x, size, 'bilinear', align_corners=False) then scale*v + shift (gifb200_resize_bilinear):
    x (B,3,H,W) fp32 with any strides -> channels-last (B,size[0],size[1],channels), channels 3.. zero."""
    _forward_only("resize_bilinear", x)
    require_cuda(x)
    B, C, H, W = x.shape
    if C != 3:
        raise ValueError(f"resize_bilinear takes (B,3,H,W) images, got {tuple(x.shape)}")
    y = torch.empty((B, size[0], size[1], channels), dtype=torch.float32, device=x.device)
    sb, sc, sh, sw = x.stride()
    check(lib.gifb200_resize_bilinear(ptr(x), ptr(y), B, H, W, sb, sc, sh, sw, size[0], size[1], channels, float(scale),
                                      float(shift), int(round_tf32), stream()), "gifb200_resize_bilinear")
    return y


def resize_bilinear_u8(x, size, channels=32, scale=1.0, shift=0.0, round_tf32=False):
    """``resize_bilinear`` of uint8 RGB images x (B,H,W,3) read as v / 255 (IEEE division) -- bitwise equal to
    ``resize_bilinear(x.permute(0,3,1,2).float() / 255)`` with a true division -- without writing that float batch
    (gifb200_resize_bilinear_u8).  Rows must be dense; the batch stride is free."""
    if not x.is_cuda:
        raise GifB200Error(f"resize_bilinear_u8 runs on CUDA tensors only; got a {x.device} tensor")
    if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != 3:
        raise ValueError(f"resize_bilinear_u8 takes uint8 (B,H,W,3) images, got {x.dtype} {tuple(x.shape)}")
    B, H, W, _ = x.shape
    if x.stride()[1:] != (3 * W, 3, 1):
        raise ValueError(f"resize_bilinear_u8: rows must be dense (strides (*, {3 * W}, 3, 1)), got {x.stride()}")
    y = torch.empty((B, size[0], size[1], channels), dtype=torch.float32, device=x.device)
    check(lib.gifb200_resize_bilinear_u8(ptr(x), ptr(y), B, H, W, x.stride(0), size[0], size[1], channels, float(scale),
                                         float(shift), int(round_tf32), stream()), "gifb200_resize_bilinear_u8")
    return y


# --------------------------------------------------------------------------------------------- layout helpers
class _BoundaryIn(torch.autograd.Function):
    """NCHW tensor coming from reference-side code -> contiguous channels-last (B,H,W,C).  Same values as ``to_nhwc``; the
    difference is the GRADIENT it hands back to the caller: contiguous in the caller's NCHW layout, as the reference's own ops
    return it (losses.py:97 does ``grad_real.view(B, -1)`` on the R1 gradient, which a permuted view would reject)."""

    @staticmethod
    def forward(ctx, x):
        return x.permute(0, 2, 3, 1).contiguous()

    @staticmethod
    def backward(ctx, g):
        return _BoundaryOut.apply(g)


class _BoundaryOut(torch.autograd.Function):
    @staticmethod
    def forward(ctx, g):
        return g.permute(0, 3, 1, 2).contiguous()

    @staticmethod
    def backward(ctx, gg):
        return _BoundaryIn.apply(gg)


def from_reference_nchw(x):
    """Entry conversion of a module-level ``forward(input)``: see _BoundaryIn.  Free (a view) when x is already a NCHW view of
    channels-last storage produced by this package."""
    if x.permute(0, 2, 3, 1).is_contiguous():
        return x.permute(0, 2, 3, 1)
    return _BoundaryIn.apply(x)


def to_nhwc(x):
    """Reference-facing NCHW tensor -> contiguous (B,H,W,C).  Free when x is an NCHW *view* of one of our outputs."""
    return _c(x.permute(0, 2, 3, 1))


def to_nchw_view(x):
    """(B,H,W,C) -> NCHW-shaped view (no copy); what the module classes return."""
    return x.permute(0, 3, 1, 2)
