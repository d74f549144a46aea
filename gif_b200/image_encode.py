"""Training images encoded on the device as the JPEGs Pillow writes: ``Image.save(f, "JPEG", quality=q)`` of an RGB image with
default options, byte for byte.  That is baseline JFIF, 4:2:0 (luma 2x2), the islow forward DCT, the quantisation tables of
JPEG Annex K scaled as libjpeg's ``jpeg_set_quality(q, force_baseline=TRUE)`` scales them, the Annex K Huffman tables, no
restart interval and no optimisation -- what the reference's ``prepare_ffhq_multiscale_dataset.py`` stores.

The encoder mirrors the decoder (image_decode.py): the host builds the headers and tables, cached per (W, H, quality),
and the kernels of csrc/jpeg_encode.cu turn a batch of images of one size into entropy-coded bytes:

    RGB->YCbCr (libjpeg fixed point) -> h2v2 downsampling -> islow FDCT + quantisation -> per-block code lengths
    -> per-image bit offsets (scan) -> bit packing (atomicOr, order-independent) -> 0xFF00 byte stuffing (count/scan/scatter)

oracle/jpeg_encode_oracle.py restates the same stages in numpy and is pinned to Pillow on the CPU."""
from functools import lru_cache
import struct

import numpy as np
import torch

from . import _lib
from .image_decode import _NATURAL

# JPEG Annex K.1, natural (row-major) order
STD_LUMA_Q = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                       14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                       49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
STD_CHROMA_Q = np.full(64, 99)
STD_CHROMA_Q.reshape(8, 8)[:4, :4] = [[17, 18, 24, 47], [18, 21, 26, 66], [24, 26, 56, 99], [47, 66, 99, 99]]

# JPEG Annex K.3: (bits[1..16], values) of the DC luma, AC luma, DC chroma and AC chroma tables
_AC_LUMA_VALS = bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a"
    "434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9"
    "aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa")
_AC_CHROMA_VALS = bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738"
    "393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5"
    "a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")
STD_HUFFMAN = (
    ((0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0), bytes(range(12))),
    ((0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125), _AC_LUMA_VALS),
    ((0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0), bytes(range(12))),
    ((0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119), _AC_CHROMA_VALS),
)
BLOCKS_PER_MCU = 6                   # Y00 Y01 Y10 Y11 Cb Cr
TABLE_INTS = 2 * 3 * 64 + 4 * 256    # per quantisation table: reciprocal, correction, shift (zigzag); 4 Huffman code tables


def quant_tables(quality):
    """libjpeg's jpeg_set_quality(quality, force_baseline=TRUE): two int32 (64,) tables in natural order."""
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return [np.clip((base * scale + 50) // 100, 1, 255).astype(np.int32) for base in (STD_LUMA_Q, STD_CHROMA_Q)]


def reciprocal(divisor):
    """libjpeg-turbo's compute_reciprocal for a 16-bit DCTELEM: (reciprocal, correction, shift) with which
    ``(|x| + correction) * reciprocal >> (16 + shift)`` is |x| / divisor rounded half up (divisor = 8 * quant, >= 8)."""
    b = divisor.bit_length() - 1
    r = 16 + b
    fq, fr = divmod(1 << r, divisor)
    c = divisor // 2
    if fr == 0:
        fq >>= 1
        r -= 1
    elif fr <= divisor // 2:
        c += 1
    else:
        fq += 1
    return fq, c, r - 16


def huffman_codes(bits, vals):
    """Canonical codes of a DHT table (JPEG Annex C): int32 (256,) entries ``length << 16 | code`` per symbol, 0 unused."""
    t = np.zeros(256, np.int32)
    code, k = 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            t[vals[k]] = ln << 16 | code
            code += 1
            k += 1
        code <<= 1
    return t


@lru_cache(maxsize=16)
def encoder_tables(quality):
    """int32 (TABLE_INTS,) for the kernels: per quantisation table (luma, chroma) reciprocal / correction / shift in
    zigzag order, then the DC0, AC0, DC1, AC1 code tables."""
    parts = []
    for q in quant_tables(quality):
        rcs = np.array([reciprocal(8 * int(v)) for v in q[_NATURAL]], np.int32)      # FDCT output is scaled by 8
        parts += [rcs[:, 0], rcs[:, 1], rcs[:, 2]]
    parts += [huffman_codes(*t) for t in STD_HUFFMAN]
    t = np.concatenate(parts).astype(np.int32)
    assert t.size == TABLE_INTS
    t.setflags(write=False)
    return t


def _segment(marker, body):
    return struct.pack(">BBH", 0xFF, marker, len(body) + 2) + body


@lru_cache(maxsize=64)
def jpeg_header(w, h, quality):
    """SOI, JFIF APP0 1.01 (no units, 1:1), two DQT, SOF0 (4:2:0), DHT DC0 AC0 DC1 AC1 -- everything before SOS, split where
    a COM segment goes (after APP0): (head, tail)."""
    if not (0 < w < 65536 and 0 < h < 65536):
        raise ValueError(f"JPEG images are at most 65535 x 65535 pixels, got {w} x {h}")
    head = b"\xff\xd8" + _segment(0xE0, b"JFIF\0\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    tail = b"".join(_segment(0xDB, bytes([i]) + q[_NATURAL].astype(np.uint8).tobytes())
                    for i, q in enumerate(quant_tables(quality)))
    tail += _segment(0xC0, struct.pack(">BHHB", 8, h, w, 3) + bytes([1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for i, (bits, vals) in enumerate(STD_HUFFMAN):
        tail += _segment(0xC4, bytes([(i & 1) << 4 | i >> 1]) + bytes(bits) + bytes(vals))
    tail += _segment(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
    return head, tail


def comment_segment(comment):
    """The COM segment Pillow writes for ``im.info["comment"]``: bytes as they are, a str (as a PNG text chunk gives it) in
    UTF-8.  Pillow cannot write a comment longer than one segment (65533 bytes), and neither can this."""
    if not comment:
        return b""
    if isinstance(comment, str):
        comment = comment.encode()
    if len(comment) > 65533:
        raise ValueError(f"a JPEG comment is at most 65533 bytes, got {len(comment)}")
    return _segment(0xFE, comment)


def jpeg_file(w, h, quality, entropy, comment=None):
    """Header (+ COM) + entropy-coded bytes (stuffed, padded) + EOI."""
    head, tail = jpeg_header(w, h, quality)
    return head + comment_segment(comment) + tail + entropy + b"\xff\xd9"


def block_layout(w, h):
    """(MCU columns, MCU rows, blocks per image) of a 4:2:0 scan."""
    mx, my = -(-w // 16), -(-h // 16)
    return mx, my, mx * my * BLOCKS_PER_MCU


def encode_jpeg_batch(x, quality=100, comments=None):
    """uint8 (B, H, W, 3) CUDA tensor of RGB images -> list of B JPEG files (bytes), each equal to what
    ``Image.fromarray(x[i]).save(f, "JPEG", quality=quality)`` writes (with ``im.info["comment"] = comments[i]`` when
    given).  All kernels run on the current stream; the byte counts come back in one small copy, then the bytes."""
    if x.dim() != 4 or x.shape[3] != 3 or x.dtype != torch.uint8 or not x.is_cuda:
        raise ValueError(f"encode_jpeg_batch: x must be a uint8 CUDA (B, H, W, 3) tensor, got {x.dtype} {tuple(x.shape)} "
                         f"on {x.device}")
    B, H, W, _ = x.shape
    if comments is not None and len(comments) != B:
        raise ValueError(f"encode_jpeg_batch: {len(comments)} comments for {B} images")
    jpeg_header(W, H, quality)                         # validates the size
    x = x.contiguous()
    dev = x.device
    tables = _tables_device(quality, dev)
    ws_bytes = int(_lib.lib.gifb200_jpeg_encode_workspace_bytes(B, H, W))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    cap = int(_lib.lib.gifb200_jpeg_encode_out_bytes(B, H, W))
    out = torch.empty(cap, dtype=torch.uint8, device=dev)
    sizes = torch.empty(B, dtype=torch.int64, device=dev)
    _lib.check(_lib.lib.gifb200_jpeg_encode(x.data_ptr(), tables.data_ptr(), B, H, W, out.data_ptr(), sizes.data_ptr(),
                                            ws.data_ptr(), ws_bytes, _lib.stream()), "jpeg_encode")
    n = sizes.cpu().tolist()
    host = torch.empty(sum(n), dtype=torch.uint8, pin_memory=True)        # pinned: a pageable copy runs at a few GB/s
    host.copy_(out[:sum(n)])
    data = host.numpy().tobytes()
    res, o = [], 0
    for i, k in enumerate(n):
        res.append(jpeg_file(W, H, quality, data[o:o + k], comments[i] if comments is not None else None))
        o += k
    return res


@lru_cache(maxsize=16)
def _tables_device(quality, device):
    return torch.from_numpy(encoder_tables(quality).copy()).to(device)
