"""The FID feature network -- pytorch_fid's InceptionV3 with the FID blocks (my_utils/pytorch_fid/inception.py:17-321) --
forward-only on the library's own kernels: gifb200_resize_bilinear (resize + 2x-1), gifb200_conv2d_ex (every BasicConv2d,
BatchNorm folded, ReLU fused, branches written straight into their slice of the block output: no torch.cat),
gifb200_pool2d and gifb200_rows_sum (the final average pool).

Weights: the FID file ``pt_inception-2015-12-05-6726825d.pth`` (torchvision key names) or a saved pytorch_fid
``InceptionV3.state_dict()`` (``blocks.i.j.*`` names), given as a path or a state dict, or found under $TORCH_HOME /
$TORCH_HOME/hub/checkpoints.  It is never downloaded.  BatchNorm (eps 0.001) is folded into the convolution on the host in
float64.  Channel counts are padded to multiples of 32 with zero weights and zero bias, so the padded channels are exactly 0
and the tensor-core kernels take every layer.  The precision follows ``ops.set_precision``."""
import hashlib
import os
import re

import torch
import torch.nn as nn

from . import ops
from ._lib import check, lib, ptr, stream

FID_WEIGHTS_FILE = "pt_inception-2015-12-05-6726825d.pth"
BN_EPS = 0.001
_HASH_REGEX = re.compile(r"-([a-f0-9]*)\.")          # torch.hub's check_hash convention


def _pad32(c):
    return (c + 31) // 32 * 32


# (name, Ci, Co, kh, kw, stride, pad_h, pad_w) of every BasicConv2d, grouped by the pytorch_fid block that owns it
def _a(p, cin, pool):
    return [(f"{p}.branch1x1", cin, 64, 1, 1, 1, 0, 0), (f"{p}.branch5x5_1", cin, 48, 1, 1, 1, 0, 0),
            (f"{p}.branch5x5_2", 48, 64, 5, 5, 1, 2, 2), (f"{p}.branch3x3dbl_1", cin, 64, 1, 1, 1, 0, 0),
            (f"{p}.branch3x3dbl_2", 64, 96, 3, 3, 1, 1, 1), (f"{p}.branch3x3dbl_3", 96, 96, 3, 3, 1, 1, 1),
            (f"{p}.branch_pool", cin, pool, 1, 1, 1, 0, 0)]


def _c(p, c7):
    return [(f"{p}.branch1x1", 768, 192, 1, 1, 1, 0, 0), (f"{p}.branch7x7_1", 768, c7, 1, 1, 1, 0, 0),
            (f"{p}.branch7x7_2", c7, c7, 1, 7, 1, 0, 3), (f"{p}.branch7x7_3", c7, 192, 7, 1, 1, 3, 0),
            (f"{p}.branch7x7dbl_1", 768, c7, 1, 1, 1, 0, 0), (f"{p}.branch7x7dbl_2", c7, c7, 7, 1, 1, 3, 0),
            (f"{p}.branch7x7dbl_3", c7, c7, 1, 7, 1, 0, 3), (f"{p}.branch7x7dbl_4", c7, c7, 7, 1, 1, 3, 0),
            (f"{p}.branch7x7dbl_5", c7, 192, 1, 7, 1, 0, 3), (f"{p}.branch_pool", 768, 192, 1, 1, 1, 0, 0)]


def _e(p, cin):
    return [(f"{p}.branch1x1", cin, 320, 1, 1, 1, 0, 0), (f"{p}.branch3x3_1", cin, 384, 1, 1, 1, 0, 0),
            (f"{p}.branch3x3_2a", 384, 384, 1, 3, 1, 0, 1), (f"{p}.branch3x3_2b", 384, 384, 3, 1, 1, 1, 0),
            (f"{p}.branch3x3dbl_1", cin, 448, 1, 1, 1, 0, 0), (f"{p}.branch3x3dbl_2", 448, 384, 3, 3, 1, 1, 1),
            (f"{p}.branch3x3dbl_3a", 384, 384, 1, 3, 1, 0, 1), (f"{p}.branch3x3dbl_3b", 384, 384, 3, 1, 1, 1, 0),
            (f"{p}.branch_pool", cin, 192, 1, 1, 1, 0, 0)]


# pytorch_fid block index -> [(module name as in blocks.i.j, its convolutions)]
BLOCKS = [
    [("Conv2d_1a_3x3", [("Conv2d_1a_3x3", 3, 32, 3, 3, 2, 0, 0)]), ("Conv2d_2a_3x3", [("Conv2d_2a_3x3", 32, 32, 3, 3, 1, 0, 0)]),
     ("Conv2d_2b_3x3", [("Conv2d_2b_3x3", 32, 64, 3, 3, 1, 1, 1)])],
    [("Conv2d_3b_1x1", [("Conv2d_3b_1x1", 64, 80, 1, 1, 1, 0, 0)]), ("Conv2d_4a_3x3", [("Conv2d_4a_3x3", 80, 192, 3, 3, 1, 0, 0)])],
    [("Mixed_5b", _a("Mixed_5b", 192, 32)), ("Mixed_5c", _a("Mixed_5c", 256, 64)), ("Mixed_5d", _a("Mixed_5d", 288, 64)),
     ("Mixed_6a", [("Mixed_6a.branch3x3", 288, 384, 3, 3, 2, 0, 0), ("Mixed_6a.branch3x3dbl_1", 288, 64, 1, 1, 1, 0, 0),
                   ("Mixed_6a.branch3x3dbl_2", 64, 96, 3, 3, 1, 1, 1), ("Mixed_6a.branch3x3dbl_3", 96, 96, 3, 3, 2, 0, 0)]),
     ("Mixed_6b", _c("Mixed_6b", 128)), ("Mixed_6c", _c("Mixed_6c", 160)), ("Mixed_6d", _c("Mixed_6d", 160)),
     ("Mixed_6e", _c("Mixed_6e", 192))],
    [("Mixed_7a", [("Mixed_7a.branch3x3_1", 768, 192, 1, 1, 1, 0, 0), ("Mixed_7a.branch3x3_2", 192, 320, 3, 3, 2, 0, 0),
                   ("Mixed_7a.branch7x7x3_1", 768, 192, 1, 1, 1, 0, 0), ("Mixed_7a.branch7x7x3_2", 192, 192, 1, 7, 1, 0, 3),
                   ("Mixed_7a.branch7x7x3_3", 192, 192, 7, 1, 1, 3, 0), ("Mixed_7a.branch7x7x3_4", 192, 192, 3, 3, 2, 0, 0)]),
     ("Mixed_7b", _e("Mixed_7b", 1280)), ("Mixed_7c", _e("Mixed_7c", 2048))],
]
_PARAMS = ("conv.weight", "bn.weight", "bn.bias", "bn.running_mean", "bn.running_var")


def default_weight_paths():
    home = os.environ.get("TORCH_HOME") or os.path.join(os.environ.get("XDG_CACHE_HOME") or os.path.expanduser("~/.cache"),
                                                        "torch")
    return [os.path.join(home, FID_WEIGHTS_FILE), os.path.join(home, "hub", "checkpoints", FID_WEIGHTS_FILE)]


def load_weights(weights=None):
    """State dict of the FID weights: ``weights`` is a state dict, a path, or None (search ``default_weight_paths()``).
    Files are loaded with ``weights_only=True`` after checking the sha256 prefix their name carries (torch hub's rule).
    Missing file: FileNotFoundError naming the paths tried; nothing is downloaded."""
    if isinstance(weights, dict):
        return weights
    paths = [os.fspath(weights)] if weights is not None else default_weight_paths()
    path = next((p for p in paths if os.path.isfile(p)), None)
    if path is None:
        raise FileNotFoundError(f"FID Inception weights ({FID_WEIGHTS_FILE}) not found; tried: {', '.join(paths)}. "
                                "gif_b200 never downloads them: place the file there or pass weights=<path or state dict>.")
    m = _HASH_REGEX.search(os.path.basename(path))
    if m and m.group(1):
        h = hashlib.sha256()
        with open(path, "rb") as f:
            for chunk in iter(lambda: f.read(1 << 20), b""):
                h.update(chunk)
        if not h.hexdigest().startswith(m.group(1)):
            raise RuntimeError(f"{path}: sha256 {h.hexdigest()[:16]}... does not start with the prefix {m.group(1)} in its name")
    return torch.load(path, map_location="cpu", weights_only=True)


def canonical_state_dict(sd, blocks=range(4)):
    """torchvision-named conv / BN tensors of the given blocks from either key layout; ``fc.*`` and ``num_batches_tracked``
    are ignored, tensors of later blocks are accepted and dropped, anything else -- or a missing tensor -- raises KeyError."""
    by_module = {}
    for bi, mods in enumerate(BLOCKS):
        for j, (mod, convs) in enumerate(mods):
            by_module[mod] = bi
            by_module[f"blocks.{bi}.{j}"] = (bi, mod)
    known = {f"{c[0]}.{p}" for mods in BLOCKS for _, convs in mods for c in convs for p in _PARAMS}
    out, unexpected = {}, []
    for k, v in sd.items():
        if k.startswith("fc.") or k.endswith("num_batches_tracked"):
            continue
        name = k
        if k.startswith("blocks."):
            head = ".".join(k.split(".")[:3])
            ent = by_module.get(head)
            name = ent[1] + k[len(head):] if isinstance(ent, tuple) else None
        if name is None or name not in known:
            unexpected.append(k)
            continue
        out[name] = v
    if unexpected:
        raise KeyError(f"FID Inception weights: unexpected keys {unexpected[:8]}{' ...' if len(unexpected) > 8 else ''}")
    need = [f"{c[0]}.{p}" for bi in blocks for _, convs in BLOCKS[bi] for c in convs for p in _PARAMS]
    missing = [k for k in need if k not in out]
    if missing:
        raise KeyError(f"FID Inception weights: missing keys {missing[:8]}{' ...' if len(missing) > 8 else ''}")
    return {k: out[k] for k in need}


def fold_bn(w, gamma, beta, mean, var, eps=BN_EPS):
    """conv (no bias) -> BatchNorm2d.eval(): weight and bias of the equivalent conv, computed in float64."""
    w, gamma, beta, mean, var = (t.detach().to(torch.float64).cpu() for t in (w, gamma, beta, mean, var))
    s = gamma / torch.sqrt(var + eps)
    return w * s[:, None, None, None], beta - mean * s


class _FoldedConv(nn.Module):
    """One BasicConv2d: folded, channel-padded tap-major weights (kh*kw, Co32, Ci32) and bias (Co32) as fp32 buffers (not in
    the state dict), plus the persistent staged workspace of gifb200_conv2d_ex (restaged when moved or when the precision
    mode changes)."""

    def __init__(self, spec, w, b):
        super().__init__()
        self.name, ci, co, self.kh, self.kw, self.stride, ph, pw = spec
        self.pad = (ph, pw)
        self.ci, self.co = _pad32(ci), _pad32(co)
        wt = torch.zeros(self.kh * self.kw, self.co, self.ci, dtype=torch.float64)
        wt[:, :co, :ci] = w.permute(2, 3, 0, 1).reshape(self.kh * self.kw, co, ci)
        bias = torch.zeros(self.co, dtype=torch.float64)
        bias[:co] = b
        self.register_buffer("weight", wt.float(), persistent=False)
        self.register_buffer("bias", bias.float(), persistent=False)
        self.ws = [None, None]

    def _apply(self, fn, recurse=True):
        self.ws = [None, None]
        return super()._apply(fn, recurse)

    def forward(self, x, out=None, c0=0):
        return ops.conv2d_ex(x, self.weight, self.kh, self.kw, self.stride, self.pad, bias=self.bias, relu=True, out=out,
                             c0=c0, round_tf32=ops.tf32_enabled(), workspace=self.ws)


class InceptionV3(nn.Module):
    """pytorch_fid.InceptionV3 (inception.py:17-164) on gif_b200 kernels, forward only: (B,3,H,W) in [0,1] (or uint8
    (B,H,W,3), see ``forward``) -> list of the requested blocks' feature maps, NCHW views of channels-last storage, sorted
    by block index."""

    DEFAULT_BLOCK_INDEX = 3
    BLOCK_INDEX_BY_DIM = {64: 0, 192: 1, 768: 2, 2048: 3}

    def __init__(self, output_blocks=(DEFAULT_BLOCK_INDEX,), resize_input=True, normalize_input=True, requires_grad=False,
                 use_fid_inception=True, weights=None):
        super().__init__()
        if not use_fid_inception:
            raise NotImplementedError("only the FID Inception weights are supported (use_fid_inception=True)")
        if requires_grad:
            raise NotImplementedError("gif_b200's InceptionV3 is forward-only (requires_grad=False)")
        self.resize_input = resize_input
        self.normalize_input = normalize_input
        self.output_blocks = sorted(output_blocks)
        self.last_needed_block = max(output_blocks)
        assert self.last_needed_block <= 3, "Last possible output block index is 3"
        sd = canonical_state_dict(load_weights(weights), range(self.last_needed_block + 1))
        self.convs = nn.ModuleDict()
        for bi in range(self.last_needed_block + 1):
            for _, convs in BLOCKS[bi]:
                for spec in convs:
                    n = spec[0]
                    w, b = fold_bn(*(sd[f"{n}.{p}"] for p in _PARAMS))
                    self.convs[n.replace(".", "__")] = _FoldedConv(spec, w, b)

    def _conv(self, name, x, out=None, c0=0):
        return self.convs[name.replace(".", "__")](x, out, c0)

    def _pool(self, x, op, stride, pad, out=None, c0=0):
        return ops.pool2d(x, op, stride, pad, out=out, c0=c0, round_tf32=ops.tf32_enabled())

    def _new(self, x, h, w, c):
        return torch.empty((x.shape[0], h, w, c), dtype=torch.float32, device=x.device)

    def _mixed_a(self, p, x, pool):
        B, H, W, _ = x.shape
        y = self._new(x, H, W, 224 + pool)
        self._conv(f"{p}.branch1x1", x, y, 0)
        self._conv(f"{p}.branch5x5_2", self._conv(f"{p}.branch5x5_1", x), y, 64)
        t = self._conv(f"{p}.branch3x3dbl_2", self._conv(f"{p}.branch3x3dbl_1", x))
        self._conv(f"{p}.branch3x3dbl_3", t, y, 128)
        self._conv(f"{p}.branch_pool", self._pool(x, "avg", 1, 1), y, 224)
        return y

    def _mixed_b(self, x):
        B, H, W, C = x.shape
        Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
        y = self._new(x, Ho, Wo, 384 + 96 + C)
        self._conv("Mixed_6a.branch3x3", x, y, 0)
        t = self._conv("Mixed_6a.branch3x3dbl_2", self._conv("Mixed_6a.branch3x3dbl_1", x))
        self._conv("Mixed_6a.branch3x3dbl_3", t, y, 384)
        self._pool(x, "max", 2, 0, y, 480)
        return y

    def _mixed_c(self, p, x):
        B, H, W, _ = x.shape
        y = self._new(x, H, W, 768)
        self._conv(f"{p}.branch1x1", x, y, 0)
        t = self._conv(f"{p}.branch7x7_2", self._conv(f"{p}.branch7x7_1", x))
        self._conv(f"{p}.branch7x7_3", t, y, 192)
        t = self._conv(f"{p}.branch7x7dbl_1", x)
        for i in (2, 3, 4):
            t = self._conv(f"{p}.branch7x7dbl_{i}", t)
        self._conv(f"{p}.branch7x7dbl_5", t, y, 384)
        self._conv(f"{p}.branch_pool", self._pool(x, "avg", 1, 1), y, 576)
        return y

    def _mixed_d(self, x):
        B, H, W, C = x.shape
        Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
        y = self._new(x, Ho, Wo, 320 + 192 + C)
        self._conv("Mixed_7a.branch3x3_2", self._conv("Mixed_7a.branch3x3_1", x), y, 0)
        t = self._conv("Mixed_7a.branch7x7x3_1", x)
        for i in (2, 3):
            t = self._conv(f"Mixed_7a.branch7x7x3_{i}", t)
        self._conv("Mixed_7a.branch7x7x3_4", t, y, 320)
        self._pool(x, "max", 2, 0, y, 512)
        return y

    def _mixed_e(self, p, x, max_pool):
        B, H, W, _ = x.shape
        y = self._new(x, H, W, 2048)
        self._conv(f"{p}.branch1x1", x, y, 0)
        t = self._conv(f"{p}.branch3x3_1", x)
        self._conv(f"{p}.branch3x3_2a", t, y, 320)
        self._conv(f"{p}.branch3x3_2b", t, y, 704)
        t = self._conv(f"{p}.branch3x3dbl_2", self._conv(f"{p}.branch3x3dbl_1", x))
        self._conv(f"{p}.branch3x3dbl_3a", t, y, 1088)
        self._conv(f"{p}.branch3x3dbl_3b", t, y, 1472)
        self._conv(f"{p}.branch_pool", self._pool(x, "max" if max_pool else "avg", 1, 1), y, 1856)
        return y

    def _block(self, i, x):
        if i == 0:
            x = self._conv("Conv2d_2b_3x3", self._conv("Conv2d_2a_3x3", self._conv("Conv2d_1a_3x3", x)))
            return self._pool(x, "max", 2, 0)
        if i == 1:
            return self._pool(self._conv("Conv2d_4a_3x3", self._conv("Conv2d_3b_1x1", x)), "max", 2, 0)
        if i == 2:
            x = self._mixed_a("Mixed_5b", x, 32)
            x = self._mixed_a("Mixed_5c", x, 64)
            x = self._mixed_a("Mixed_5d", x, 64)
            x = self._mixed_b(x)
            for p in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
                x = self._mixed_c(p, x)
            return x
        x = self._mixed_e("Mixed_7c", self._mixed_e("Mixed_7b", self._mixed_d(x), False), True)
        B, H, W, C = x.shape                                     # adaptive average pool to 1x1: sum over pixels, scale
        s = torch.empty((B, C), dtype=torch.float32, device=x.device)
        check(lib.gifb200_rows_sum(ptr(x), ptr(s), B, H * W, C, stream()), "gifb200_rows_sum")
        check(lib.gifb200_axpby(ptr(s), None, ptr(s), s.numel(), 1.0 / (H * W), 0.0, 0, stream()), "gifb200_axpby")
        return s.view(B, 1, 1, C)

    def forward(self, inp):
        """``inp``: (B,3,H,W) float32 in [0,1], or uint8 RGB (B,H,W,3) on the device, read as v / 255 by the input resize
        (``ops.resize_bilinear_u8``: fid_score.py:106-112's float batch without materialising it)."""
        if torch.is_grad_enabled() and inp.requires_grad:
            raise RuntimeError("gif_b200's InceptionV3 is forward-only: the input must not require grad")
        u8 = inp.dtype == torch.uint8
        H, W = (299, 299) if self.resize_input else tuple(inp.shape[1:3] if u8 else inp.shape[2:])
        scale, shift = (2.0, -1.0) if self.normalize_input else (1.0, 0.0)
        resize = ops.resize_bilinear_u8 if u8 else ops.resize_bilinear
        x = resize(inp, (H, W), 32, scale, shift, round_tf32=ops.tf32_enabled())
        outp = []
        for i in range(self.last_needed_block + 1):
            x = self._block(i, x)
            if i in self.output_blocks:
                outp.append(x.permute(0, 3, 1, 2))
        return outp
