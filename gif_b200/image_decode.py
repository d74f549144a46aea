"""Training images decoded on the device, bit-exact with Pillow (SURVEY 8f.3).

The host does only what is cheap or inherently serial: it parses JPEG markers and PNG chunks, builds the Huffman and
quantisation tables, removes JPEG byte stuffing and splits the scan at restart markers, checks PNG CRCs and inflates the
IDAT stream with zlib (which releases the GIL).  ``host_decode`` does this for one image and names it in every error it
raises.  ``DecodeBatch`` packs a batch of such images, JPEG and PNG in any mix, into one pinned arena (``JpegBatch`` /
``PngBatch`` lay out each kind), so a batch costs one host-to-device copy, and runs the kernels of csrc/image_decode.cu
on it; ``check_status`` turns their per-image status words into an ``UnsupportedImage`` naming the image:

    JPEG  parallel entropy decode -> dequantise + islow IDCT -> fancy upsampling + YCbCr->RGB       (libjpeg-turbo defaults)
    PNG   scanline unfiltering (None/Sub/Up/Average/Paeth) -> RGB (grey replicated, alpha dropped)  (``convert("RGB")``)
    resize Pillow's two-pass bicubic / Lanczos with 22-bit fixed-point weights                        (``Image.resize``)
    unit  (v / 255 - 0.5) / 0.5 into NCHW slices                                                      (ToTensor + Normalize)

Anything outside the supported subset raises ``UnsupportedImage`` naming the reason; ``data.decode_image`` (PIL) remains
the path for such files."""
import math
import re
import struct
import zlib
from functools import lru_cache
from typing import NamedTuple

import numpy as np
import torch

from . import _lib

# Entropy-coded bytes per decoding thread.  A run from a guessed state needs several blocks to fall into step with the
# true decode (bit position, coefficient index AND the block's place in the MCU, which selects the Huffman tables), and a
# quality-100 block is ~75 bytes; shorter chunks mean more threads and less bit-serial work per pass.
CHUNK_BYTES = 1024
DESC_INTS, SEG_INTS, HUFF_INTS, PNG_DESC_INTS = 48, 8, 804, 8
# descriptor field offsets (csrc/image_decode.cuh JpegDesc)
JD_W, JD_H, JD_NCOMP, JD_HMAX, JD_VMAX, JD_MCUX, JD_MCUY, JD_BPM, JD_BLOCK_BASE, JD_NBLOCKS, JD_OUT_OFF = range(11)
JD_H0, JD_V0, JD_BW0, JD_CBASE0, JD_DCT0, JD_ACT0, JD_BLK0 = 11, 14, 17, 20, 23, 26, 29
STATUS_BAD_CODE, STATUS_BLOCK_COUNT, STATUS_PNG_FILTER = 1, 2, 4

_NATURAL = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7,
                     14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39,
                     46, 53, 60, 61, 54, 47, 55, 62, 63])


class UnsupportedImage(ValueError):
    """The encoded image is malformed or outside what the device decoders support."""


# ------------------------------------------------------------------------------------------------------------------ JPEG
_SOF_NAMES = {0xC2: "progressive JPEG", 0xC3: "lossless JPEG", 0xC5: "hierarchical JPEG", 0xC6: "hierarchical JPEG",
              0xC7: "hierarchical JPEG", 0xC9: "arithmetic-coded JPEG", 0xCA: "progressive arithmetic-coded JPEG",
              0xCB: "lossless arithmetic-coded JPEG", 0xCD: "hierarchical JPEG", 0xCE: "hierarchical JPEG",
              0xCF: "hierarchical JPEG"}


@lru_cache(maxsize=256)
def huffman_table(bits, vals):
    """int32[HUFF_INTS] device table of a DHT table: 9-bit lookahead (len << 8 | symbol), maxcode[18], valoff[18], vals[256]
    (canonical code assignment, JPEG Annex C; the code-space check of libjpeg's jpeg_make_d_derived_tbl)."""
    t = np.zeros(HUFF_INTS, np.int32)
    t[512:530] = -1
    code, k = 0, 0
    for l in range(1, 17):
        n = bits[l - 1]
        if n:
            t[530 + l] = k - code
            for _ in range(n):
                if l <= 9:
                    s = code << (9 - l)
                    t[s:s + (1 << (9 - l))] = (l << 8) | vals[k]
                code += 1
                k += 1
            t[512 + l] = code - 1
        if code >= (1 << l):            # also rejects a code of all ones, which JPEG reserves
            raise UnsupportedImage("bad Huffman table (code space overflow)")
        code <<= 1
    t[548:548 + len(vals)] = vals
    t.setflags(write=False)
    return t


def parse_jpeg(data):
    """Markers of a baseline JPEG -> dict with the frame, tables and the un-stuffed entropy-coded segments.  Raises
    ``UnsupportedImage`` for progressive / arithmetic / lossless / 12-bit / CMYK / Adobe-RGB / multi-scan files and for
    headers that are truncated or inconsistent."""
    try:
        return _parse_jpeg(data)
    except (IndexError, ValueError) as e:
        if isinstance(e, UnsupportedImage):
            raise
        raise UnsupportedImage(f"corrupt JPEG header (a marker segment is shorter than its contents: {e})") from None


def _parse_jpeg(data):
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise UnsupportedImage("not a JPEG file (no SOI marker)")
    pos, qt, ht, frame, dri, adobe, jfif = 2, {}, {}, None, 0, None, False
    while True:
        while pos < n and data[pos] == 0xFF and pos + 1 < n and data[pos + 1] == 0xFF:
            pos += 1                                   # fill bytes
        if pos + 4 > n:
            raise UnsupportedImage("truncated JPEG header")
        if data[pos] != 0xFF:
            raise UnsupportedImage(f"corrupt JPEG: expected a marker at byte {pos}")
        m = data[pos + 1]
        ln = (data[pos + 2] << 8) | data[pos + 3]
        seg = data[pos + 4:pos + 2 + ln]
        if ln < 2 or pos + 2 + ln > n:
            raise UnsupportedImage("truncated JPEG header")
        if m in _SOF_NAMES:
            raise UnsupportedImage(f"{_SOF_NAMES[m]} is not supported (baseline only)")
        if m in (0xC0, 0xC1):
            p, h, w, nc = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if p != 8:
                raise UnsupportedImage(f"{p}-bit JPEG is not supported (8-bit only)")
            if nc not in (1, 3):
                raise UnsupportedImage(f"{nc}-component JPEG (CMYK?) is not supported (1 or 3 components)")
            if h == 0 or w == 0:
                raise UnsupportedImage("JPEG without a height in its frame header (DNL) is not supported")
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nc)]
            frame = (w, h, comps)
        elif m == 0xC4:
            o = 0
            while o < len(seg):
                tc, th = seg[o] >> 4, seg[o] & 15
                bits = tuple(seg[o + 1:o + 17])
                cnt = sum(bits)
                vals = tuple(seg[o + 17:o + 17 + cnt])
                if tc > 1 or th > 1 or len(vals) != cnt or cnt > 256:
                    raise UnsupportedImage("bad or unsupported Huffman table")
                if tc == 0 and any(v > 15 for v in vals):
                    raise UnsupportedImage("bad DC Huffman table")
                ht[(tc, th)] = (bits, vals)
                o += 17 + cnt
        elif m == 0xDB:
            o = 0
            while o < len(seg):
                pq, tq = seg[o] >> 4, seg[o] & 15
                if pq == 0:
                    q = np.frombuffer(seg[o + 1:o + 65], np.uint8).astype(np.int32)
                    o += 65
                else:
                    q = np.frombuffer(seg[o + 1:o + 129], ">u2").astype(np.int32)
                    o += 129
                if q.size != 64 or tq > 3:
                    raise UnsupportedImage("bad quantisation table")
                nat = np.empty(64, np.int32)
                nat[_NATURAL] = q
                qt[tq] = nat
        elif m == 0xDD:
            dri = (seg[0] << 8) | seg[1]
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            adobe = seg[11]
        elif m == 0xE0 and seg[:5] == b"JFIF\0":
            jfif = True
        elif m == 0xDA:
            if frame is None:
                raise UnsupportedImage("JPEG scan before its frame header")
            ns = seg[0]
            if ns != len(frame[2]):
                raise UnsupportedImage("multi-scan (non-interleaved) baseline JPEG is not supported")
            ids = [c[0] for c in frame[2]]
            tables = {}
            for i in range(ns):
                cid, tt = seg[1 + 2 * i], seg[2 + 2 * i]
                if cid not in ids:
                    raise UnsupportedImage("JPEG scan names an unknown component")
                tables[cid] = (tt >> 4, tt & 15)
            return _finish_jpeg(data, pos + 2 + ln, frame, qt, ht, tables, dri, adobe, jfif)
        elif m == 0xD9:
            raise UnsupportedImage("JPEG without a scan")
        pos += 2 + ln


def _finish_jpeg(data, start, frame, qt, ht, tables, dri, adobe, jfif):
    w, h, comps = frame
    nc = len(comps)
    if nc == 3:
        rgb = (adobe == 0) if (not jfif and adobe is not None) else (not jfif and [c[0] for c in comps] == [82, 71, 66])
        if rgb:
            raise UnsupportedImage("JPEG with an RGB (Adobe transform 0) colour space is not supported")
        hs, vs = comps[0][1], comps[0][2]
        if (hs, vs) not in ((1, 1), (2, 1), (1, 2), (2, 2)) or any(c[1:3] != (1, 1) for c in comps[1:]):
            raise UnsupportedImage(f"JPEG sampling {[c[1:3] for c in comps]} is not supported (luma 1x1/2x1/1x2/2x2, chroma 1x1)")
        mcux, mcuy = -(-w // (8 * hs)), -(-h // (8 * vs))
        blk = [(ci, dx, dy) for ci, c in enumerate(comps) for dy in range(c[2]) for dx in range(c[1])]
        bw = [mcux * c[1] for c in comps]
        bh = [mcuy * c[2] for c in comps]
    else:
        hs = vs = 1
        mcux, mcuy = -(-w // 8), -(-h // 8)
        blk, bw, bh = [(0, 0, 0)], [mcux], [mcuy]
    q = []
    for c in comps:
        if c[3] not in qt:
            raise UnsupportedImage("JPEG component uses an undefined quantisation table")
        q.append(qt[c[3]])
    huff = np.zeros((4, HUFF_INTS), np.int32)
    used = [tables[c[0]] for c in comps]
    for cls in (0, 1):
        for th in (0, 1):
            if any(u[cls] == th for u in used):
                if (cls, th) not in ht:
                    raise UnsupportedImage("JPEG scan uses an undefined Huffman table")
                huff[cls * 2 + th] = huffman_table(*ht[(cls, th)])
    segs, truncated = _entropy_segments(data, start)
    n_mcu = mcux * mcuy
    n_seg = -(-n_mcu // dri) if dri else 1
    if len(segs) > n_seg:
        raise UnsupportedImage(f"JPEG has {len(segs)} restart intervals, its header implies {n_seg}")
    segs += [b""] * (n_seg - len(segs))                      # missing intervals: the device reports the image
    return {"w": w, "h": h, "ncomp": nc, "hs": hs, "vs": vs, "mcux": mcux, "mcuy": mcuy, "blk": blk, "bw": bw, "bh": bh,
            "q": q, "huff": huff, "dc": [u[0] for u in used], "ac": [u[1] for u in used], "dri": dri or n_mcu,
            "segments": segs, "truncated": truncated}


_END_MARKER = re.compile(rb"\xff[^\x00\xd0-\xd7\xff]")
_RST_OR_FILL = re.compile(rb"\xff[\xd0-\xd7\xff]")


def _entropy_segments(data, start):
    """Entropy-coded data after SOS -> list of un-stuffed segments (split at RSTn), and whether no end marker was found."""
    m = _END_MARKER.search(data, start)
    if m is not None and _RST_OR_FILL.search(data, start, m.start()) is None:
        return [data[start:m.start()].replace(b"\xff\x00", b"\xff")], False     # one segment, stuffing only
    a = np.frombuffer(data, np.uint8)[start:]
    ff = np.flatnonzero(a[:-1] == 0xFF)
    nxt = a[ff + 1]
    stop = np.flatnonzero((nxt != 0) & (nxt != 0xFF) & ((nxt < 0xD0) | (nxt > 0xD7)))
    end, truncated = (int(ff[stop[0]]), False) if stop.size else (len(a) - (1 if len(a) and a[-1] == 0xFF else 0), True)
    keep = ff < end
    ff, nxt = ff[keep], nxt[keep]
    drop = np.zeros(end, bool)
    drop[ff[nxt == 0] + 1] = True                          # stuffed zero after 0xFF
    drop[ff[nxt == 0xFF]] = True                           # fill bytes
    rst = ff[(nxt >= 0xD0) & (nxt <= 0xD7)]
    drop[rst] = True
    drop[np.minimum(rst + 1, end - 1)] = True
    body = a[:end]
    cuts = [0] + list(rst) + [end]
    return [body[lo:hi][~drop[lo:hi]].tobytes() for lo, hi in zip(cuts[:-1], cuts[1:])], truncated


class JpegBatch:
    """Parsed JPEGs packed for one ``gifb200_jpeg_decode`` call: ``data`` (uint8, the segments), ``ints`` (int32:
    descriptors, segments, chunk map, quantisation and Huffman tables), the output layout and the workspace size."""

    def __init__(self, parsed, chunk_bytes=CHUNK_BYTES):
        self.chunk_bytes = chunk_bytes
        desc = np.zeros((len(parsed), DESC_INTS), np.int32)
        seg_rows, chunk_seg, blobs, qt, ht = [], [], [], [], []
        off = out_off = blocks = n_chunk = 0
        self.shapes, self.out_offsets = [], []
        for i, p in enumerate(parsed):
            nblk = sum(bw * bh for bw, bh in zip(p["bw"], p["bh"]))
            d = desc[i]
            d[:JD_H0] = [p["w"], p["h"], p["ncomp"], p["hs"], p["vs"], p["mcux"], p["mcuy"], len(p["blk"]), blocks, nblk,
                         out_off]
            nc = p["ncomp"]
            cbase = np.concatenate([[0], np.cumsum([bw * bh for bw, bh in zip(p["bw"], p["bh"])])])[:nc]
            d[JD_H0:JD_H0 + nc] = [1 if nc == 1 else (p["hs"] if c == 0 else 1) for c in range(nc)]
            d[JD_V0:JD_V0 + nc] = [1 if nc == 1 else (p["vs"] if c == 0 else 1) for c in range(nc)]
            d[JD_BW0:JD_BW0 + nc] = p["bw"]
            d[JD_CBASE0:JD_CBASE0 + nc] = cbase
            d[JD_DCT0:JD_DCT0 + nc] = p["dc"]
            d[JD_ACT0:JD_ACT0 + nc] = p["ac"]
            d[JD_BLK0:JD_BLK0 + len(p["blk"])] = [ci | dx << 4 | dy << 8 for ci, dx, dy in p["blk"]]
            n_mcu = p["mcux"] * p["mcuy"]
            for s, seg in enumerate(p["segments"]):
                nch = max(1, -(-len(seg) // chunk_bytes))
                first = s * p["dri"]
                seg_rows.append([i, off, len(seg), first, min(p["dri"], n_mcu - first), n_chunk, nch, 0])
                chunk_seg += [len(seg_rows) - 1] * nch
                n_chunk += nch
                blobs.append(seg)
                off += len(seg)
            q = np.zeros((3, 64), np.int32)
            q[:nc] = p["q"]
            qt.append(q)
            ht.append(p["huff"])
            self.shapes.append((p["h"], p["w"]))
            self.out_offsets.append(out_off)
            blocks += nblk
            out_off += p["w"] * p["h"] * 3
        if out_off >= 2 ** 31 or off >= 2 ** 31:
            raise UnsupportedImage("JPEG batch too large for 32-bit offsets")
        self.n_img, self.n_seg, self.n_chunk, self.n_blocks = len(parsed), len(seg_rows), n_chunk, blocks
        self.max_blocks = int(desc[:, JD_NBLOCKS].max())
        self.out_bytes = out_off
        self.data = b"".join(blobs)
        seg = np.asarray(seg_rows, np.int32).reshape(-1, SEG_INTS)
        parts = [desc.ravel(), seg.ravel(), np.asarray(chunk_seg, np.int32), np.concatenate(qt).ravel(),
                 np.concatenate(ht).ravel()]
        self.int_offsets = np.concatenate([[0], np.cumsum([x.size for x in parts])])
        self.ints = np.concatenate(parts).astype(np.int32)
        self.workspace_bytes = int(_lib.lib.gifb200_jpeg_workspace_bytes(self.n_chunk, self.n_seg, self.n_blocks))

    def launch(self, data_dev, ints_dev, out, status, workspace):
        """Enqueue the decode on the current stream; data_dev / ints_dev hold ``data`` / ``ints`` on the device."""
        io = [ints_dev.data_ptr() + 4 * int(o) for o in self.int_offsets[:5]]
        _lib.check(_lib.lib.gifb200_jpeg_decode(data_dev.data_ptr(), *io, self.n_img, self.n_seg, self.n_chunk, self.n_blocks,
                                                self.max_blocks, self.chunk_bytes, out.data_ptr(), status.data_ptr(), workspace.data_ptr(),
                                                workspace.numel(), _lib.stream()), "jpeg_decode")


# ------------------------------------------------------------------------------------------------------------------- PNG
_PNG_SIG = b"\x89PNG\r\n\x1a\n"
_PNG_BPP = {0: 1, 2: 3, 6: 4}


def parse_png(data):
    """PNG chunks -> (W, H, bytes per pixel, concatenated IDAT data).  Checks every chunk CRC.  Raises ``UnsupportedImage``
    for palette, 16-bit, sub-byte, grey+alpha and interlaced images and for truncated or corrupt files."""
    try:
        return _parse_png(data)
    except struct.error as e:
        raise UnsupportedImage(f"corrupt PNG (a chunk is shorter than its contents: {e})") from None


def _parse_png(data):
    if data[:8] != _PNG_SIG:
        raise UnsupportedImage("not a PNG file (bad signature)")
    pos, n, hdr, idat = 8, len(data), None, []
    while True:
        if pos + 12 > n:
            raise UnsupportedImage("truncated PNG (no IEND chunk)")
        ln, typ = struct.unpack_from(">I4s", data, pos)
        if pos + 12 + ln > n:
            raise UnsupportedImage(f"truncated PNG ({typ.decode('latin-1')} chunk runs past the end)")
        body = data[pos + 8:pos + 8 + ln]
        if zlib.crc32(body, zlib.crc32(typ)) != struct.unpack_from(">I", data, pos + 8 + ln)[0]:
            raise UnsupportedImage(f"PNG {typ.decode('latin-1')} chunk fails its CRC")
        if typ == b"IHDR":
            w, h, depth, ct, comp, filt, inter = struct.unpack(">IIBBBBB", body)
            if ct == 3:
                raise UnsupportedImage("palette PNG is not supported")
            if depth != 8:
                raise UnsupportedImage(f"{depth}-bit PNG is not supported (8-bit only)")
            if ct not in _PNG_BPP:
                raise UnsupportedImage(f"PNG colour type {ct} is not supported (grey, RGB, RGBA)")
            if inter:
                raise UnsupportedImage("interlaced PNG is not supported")
            if comp or filt:
                raise UnsupportedImage("unknown PNG compression or filter method")
            hdr = (w, h, _PNG_BPP[ct])
        elif typ == b"IDAT":
            idat.append(body)
        elif typ == b"IEND":
            break
        pos += 12 + ln
    if hdr is None or not idat:
        raise UnsupportedImage("PNG without IHDR or IDAT")
    return hdr + (b"".join(idat),)


def inflate_png(parsed):
    """zlib-inflate the IDAT stream of ``parse_png``'s result; its size must be H rows of (1 + W * bpp) bytes."""
    w, h, bpp, z = parsed
    try:
        raw = zlib.decompress(z)
    except zlib.error as e:
        raise UnsupportedImage(f"corrupt PNG data stream ({e})") from None
    if len(raw) != h * (1 + w * bpp):
        raise UnsupportedImage(f"PNG data stream has {len(raw)} bytes, a {w}x{h} image needs {h * (1 + w * bpp)}")
    return raw


class PngBatch:
    """Inflated PNGs packed for one ``gifb200_png_unfilter`` call."""

    def __init__(self, headers, raws):
        desc = np.zeros((len(raws), PNG_DESC_INTS), np.int32)
        off = out_off = 0
        self.shapes, self.out_offsets = [], []
        for i, ((w, h, bpp, _), raw) in enumerate(zip(headers, raws)):
            desc[i, :5] = [off, w, h, bpp, out_off]
            self.shapes.append((h, w))
            self.out_offsets.append(out_off)
            off += len(raw)
            out_off += w * h * 3
        if out_off >= 2 ** 31 or off >= 2 ** 31:
            raise UnsupportedImage("PNG batch too large for 32-bit offsets")
        self.n_img, self.out_bytes, self.desc = len(raws), out_off, desc
        self.max_pixels = max(h * w for h, w in self.shapes)
        self.data_bytes = off

    def launch(self, data_dev, desc_dev, out, status):
        _lib.check(_lib.lib.gifb200_png_unfilter(data_dev.data_ptr(), desc_dev.data_ptr(), self.n_img, self.max_pixels,
                                                 out.data_ptr(), status.data_ptr(), _lib.stream()), "png_unfilter")


# --------------------------------------------------------------------------------------------------------------- batches
class HostImage(NamedTuple):
    """One image after ``host_decode``: its name (a path or a key), "jpeg" or "png", its size, bytes per pixel (JPEG
    components, PNG channels) and what the device needs: ``parse_jpeg``'s result, or the inflated PNG scanlines."""
    name: str
    kind: str
    w: int
    h: int
    bpp: int
    data: object


def host_decode(data, name):
    """The host half of decoding one encoded image, dispatched on its magic bytes as ``Image.open`` does: a baseline JPEG
    is parsed, a PNG parsed and inflated.  Every ``UnsupportedImage`` it raises starts with ``name``."""
    try:
        if data[:8] == _PNG_SIG:
            hdr = parse_png(data)
            return HostImage(name, "png", *hdr[:3], inflate_png(hdr))
        if data[:3] == b"\xff\xd8\xff":
            p = parse_jpeg(data)
            return HostImage(name, "jpeg", p["w"], p["h"], p["ncomp"], p)
        raise UnsupportedImage("not a PNG or baseline JPEG file (the device decoders read only these)")
    except UnsupportedImage as e:
        raise UnsupportedImage(f"{name}: {e}") from None


class DecodeBatch:
    """``host_decode`` results, JPEG and PNG in any mix, packed for one decode: the JPEG data, the JPEG int tables, the PNG
    scanlines and the PNG descriptors in one host arena, 256-byte aligned sections, pinned when CUDA is available.  The
    output buffer and the status words hold the JPEGs, then the PNGs, each kind in input order: ``order`` lists the input
    indices and ``names`` the images' names in that order."""

    def __init__(self, images, chunk_bytes=CHUNK_BYTES):
        self.order = sorted(range(len(images)), key=lambda i: images[i].kind == "png")      # stable: JPEGs, then PNGs
        self.names = [images[i].name for i in self.order]
        jpegs, pngs = [im for im in images if im.kind == "jpeg"], [im for im in images if im.kind == "png"]
        jb = self.jpeg = JpegBatch([im.data for im in jpegs], chunk_bytes) if jpegs else None
        pb = self.png = PngBatch([(im.w, im.h, im.bpp, b"") for im in pngs], [im.data for im in pngs]) if pngs else None
        starts = np.cumsum([0] + [im.w * im.h * 3 for im in jpegs + pngs])            # the images back to back
        self.out_bytes, self.png_out = int(starts[-1]), int(starts[len(jpegs)])
        self.views = [None] * len(images)                                              # input order
        for k, i in enumerate(self.order):
            self.views[i] = (int(starts[k]), images[i].h, images[i].w)
        sections = [[jb.data] if jb else [], [im.data for im in pngs], [jb.ints] if jb else [], [pb.desc] if pb else []]
        sections = [[np.frombuffer(b, np.uint8) for b in s] for s in sections]
        self.offsets = np.cumsum([0] + [-(-sum(b.size for b in s) // 256) * 256 for s in sections])
        self.arena = torch.empty(int(self.offsets[-1]), dtype=torch.uint8, pin_memory=torch.cuda.is_available())
        a = self.arena.numpy()
        for o, s in zip(self.offsets, sections):
            for b in s:
                a[o:o + b.size] = b
                o += b.size

    def decode(self, device, status=None):
        """Enqueue one non-blocking copy of the arena and the decode kernels on the current stream.  Returns (images,
        status): uint8 (H, W, 3) device views in input order, equal to ``np.asarray(Image.open(b).convert("RGB"))``, and
        int32 device status words in ``order`` (0 = decoded; otherwise STATUS_* bits: corrupt or truncated data), written
        to ``status`` (zeroed, one word per image) when the caller passes one."""
        d = self.arena.to(device, non_blocking=True)      # the host allocator keeps the arena until this copy has run
        sec = [d[int(lo):int(hi)] for lo, hi in zip(self.offsets[:-1], self.offsets[1:])]
        out = torch.empty(self.out_bytes, dtype=torch.uint8, device=device)
        status = torch.zeros(len(self.order), dtype=torch.int32, device=device) if status is None else status
        if self.jpeg:
            ws = torch.empty(self.jpeg.workspace_bytes, dtype=torch.uint8, device=device)
            self.jpeg.launch(sec[0], sec[2], out, status, ws)
        if self.png:
            self.png.launch(sec[1], sec[3], out[self.png_out:], status[len(self.order) - self.png.n_img:])
        return [out[o:o + h * w * 3].view(h, w, 3) for o, h, w in self.views], status


def check_status(status, names):
    """Raise ``UnsupportedImage`` naming the first image whose status word is nonzero and counting the others.
    ``status``: host-side words, one per name."""
    st = np.asarray(status)
    bad = np.flatnonzero(st)
    if bad.size:
        s = int(st[bad[0]])
        what = "corrupt PNG scanlines (unknown filter type)" if s & STATUS_PNG_FILTER else "corrupt or truncated JPEG data"
        raise UnsupportedImage(f"{names[bad[0]]}: {what} (device status {s})"
                               + (f", and {bad.size - 1} more images" if bad.size > 1 else ""))


def decode_images(blobs, device=None, chunk_bytes=CHUNK_BYTES):
    """Decode encoded images (baseline JPEG; 8-bit grey, RGB or RGBA PNG) on the device, through ``DecodeBatch``.  Returns
    (images, status) as ``DecodeBatch.decode`` does, but with the status words in input order."""
    batch = DecodeBatch([host_decode(b, f"image {i}") for i, b in enumerate(blobs)], chunk_bytes)
    images, status = batch.decode(torch.device(device or "cuda"))
    return images, status[torch.as_tensor(np.argsort(batch.order), device=status.device)]


decode_jpeg_batch = decode_png_batch = decode_images       # the names of the former per-format decoders


def as_batch(images):
    """Same-shape uint8 (H, W, 3) images -> (n, H, W, 3): a view when they lie back to back in one buffer (a run of one
    kind in ``DecodeBatch.decode``'s output), else a stacked copy."""
    x = images[0]
    step = x.numel()
    if all(y.shape == x.shape and y.is_contiguous() and y.untyped_storage().data_ptr() == x.untyped_storage().data_ptr()
           and y.data_ptr() == x.data_ptr() + k * step for k, y in enumerate(images)):
        return x.as_strided((len(images),) + tuple(x.shape), (step,) + x.stride())
    return torch.stack(images)


def shape_groups(images):
    """Images of one batch grouped by shape, in sorted shape order: [(input indices, uint8 (n, H, W, 3) ``as_batch``)]."""
    groups = {}
    for i, x in enumerate(images):
        groups.setdefault(tuple(x.shape), []).append(i)
    return [(idx, as_batch([images[i] for i in idx])) for _, idx in sorted(groups.items())]


def prefetch(pool, load, batches):
    """Yield ``[load(x) for x in batch]`` for each batch in turn.  The loads run on ``pool``; the next batch's are submitted
    when this one is taken, so they run while the caller works on this one."""
    futures = [pool.submit(load, x) for x in batches[0]] if batches else []
    for nxt in list(batches[1:]) + [[]]:
        done = [f.result() for f in futures]
        futures = [pool.submit(load, x) for x in nxt]
        yield done


# ---------------------------------------------------------------------------------------------------------------- resize
def _bicubic(x):
    x = abs(x)
    if x < 1.0:
        return ((-0.5 + 2.0) * x - (-0.5 + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * -0.5
    return 0.0


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    """Pillow's truncated sinc (lanczos_filter), through the C library's sin as Pillow calls it, one value at a time."""
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


def _resample_coeffs(filt, support, in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc (the filter's support widened by the scale when downscaling), in
    float64: int32 (out_size, ks + 2) rows [first tap, tap count, 22-bit weights...]."""
    scale = in_size / out_size
    fscale = max(scale, 1.0)
    support = support * fscale
    ks = int(np.ceil(support)) * 2 + 1
    out = np.zeros((out_size, ks + 2), np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        ss = 1.0 / fscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [filt((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        tot = sum(w)
        w = [v / tot if tot != 0.0 else v for v in w]
        out[xx, 0], out[xx, 1] = xmin, xmax
        out[xx, 2:2 + xmax] = [int(-0.5 + v * (1 << 22)) if v < 0 else int(0.5 + v * (1 << 22)) for v in w]
    out.setflags(write=False)
    return out


@lru_cache(maxsize=64)
def bicubic_coeffs(in_size, out_size):
    """``_resample_coeffs`` of Pillow's bicubic filter (support 2)."""
    return _resample_coeffs(_bicubic, 2.0, in_size, out_size)


@lru_cache(maxsize=64)
def lanczos_coeffs(in_size, out_size):
    """``_resample_coeffs`` of Pillow's Lanczos filter (support 3)."""
    return _resample_coeffs(_lanczos, 3.0, in_size, out_size)


@lru_cache(maxsize=64)
def _coeffs_device(coeffs, W, H, Wo, Ho, device):
    """Both passes' coefficients on the device, uploaded once per shape: a per-call upload would wait for the stream (a
    blocking host-to-device copy) and stall a pipeline that keeps the device busy.  A pass whose axis keeps its size is
    skipped, as Pillow skips it: its table is empty and its tap count 0."""
    ch = coeffs(W, Wo) if W != Wo else np.zeros((0, 2), np.int32)
    cv = coeffs(H, Ho) if H != Ho else np.zeros((0, 2), np.int32)
    t = torch.from_numpy(np.concatenate([ch.ravel(), cv.ravel(), [0]]).astype(np.int32)).to(device)
    return t, ch.size, ch.shape[1] - 2, cv.shape[1] - 2


def _resize_u8(coeffs, x, Ho, Wo, tmp, out, name):
    squeeze = x.dim() == 3
    xb = x.unsqueeze(0) if squeeze else x
    B, H, W, _ = xb.shape
    coef, n_h, ks_h, ks_v = _coeffs_device(coeffs, W, H, Wo, Ho, x.device)
    if tmp is None and ks_h and ks_v:
        tmp = torch.empty(B, H, Wo, 3, dtype=torch.uint8, device=x.device)
    out = torch.empty(B, Ho, Wo, 3, dtype=torch.uint8, device=x.device) if out is None else out
    _lib.check(_lib.lib.gifb200_resize_bicubic_u8(xb.contiguous().data_ptr(), tmp.data_ptr() if tmp is not None else None,
                                                  out.data_ptr(), coef.data_ptr() if ks_h else None,
                                                  coef.data_ptr() + 4 * n_h if ks_v else None, B, H, W, Ho, Wo, ks_h, ks_v,
                                                  _lib.stream()), name)
    return out[0] if squeeze else out


def resize_bicubic_u8(x, size, tmp=None, out=None):
    """uint8 (B, H, W, 3) or (H, W, 3) CUDA tensor -> (B, size, size, 3): Pillow's ``Image.resize((size, size))`` (bicubic),
    bit for bit."""
    return _resize_u8(bicubic_coeffs, x, size, size, tmp, out, "resize_bicubic_u8")


def resize_lanczos_u8(x, size, tmp=None, out=None):
    """uint8 (B, H, W, 3) or (H, W, 3) CUDA tensor -> (B, Ho, Wo, 3) for ``size`` = (Ho, Wo): Pillow's
    ``Image.resize((Wo, Ho), Image.LANCZOS)``, bit for bit."""
    Ho, Wo = size
    return _resize_u8(lanczos_coeffs, x, Ho, Wo, tmp, out, "resize_lanczos_u8")


def resized_crop_box(w, h, size):
    """torchvision's ``resize(img, size)`` (an int: the short side becomes ``size``, the long side ``int(size * long /
    short)``; an image already of that size is left alone) then ``center_crop(size)``, for a PIL image of w x h:
    ((resized w, resized h), (left, top)) of the crop.  Rounding of the offset is Python's (halves to even), as there."""
    if w <= h:
        rw, rh = size, int(size * h / w)
    else:
        rw, rh = int(size * w / h), size
    return (rw, rh), (int(round((rw - size) / 2.0)), int(round((rh - size) / 2.0)))


def u8_to_unit(x, out):
    """uint8 (B, H, W, 3) -> ``out`` (a (B, 3, H, W) float32 view, possibly a channel slice of a wider NCHW batch):
    (v / 255 - 0.5) / 0.5 as ToTensor + Normalize((0.5,)*3, (0.5,)*3) compute it."""
    B, H, W, _ = x.shape
    if out.shape != (B, 3, H, W) or out.stride()[1:] != (H * W, W, 1) or out.dtype != torch.float32:
        raise ValueError("u8_to_unit: out must be a float32 (B, 3, H, W) view with dense channel planes")
    _lib.check(_lib.lib.gifb200_u8_to_unit(x.data_ptr(), out.data_ptr(), B, H, W, out.stride(0), _lib.stream()), "u8_to_unit")
    return out


def image_to_u8(x, out=None):
    """float32 (B, 3, H, W) CUDA view with any strides (the generator's NCHW view of channels-last storage included) ->
    uint8 (B, H, W, 3): the bytes the reference's sampling scripts save, ``uint8(clip((clamp(x, -1, 1) + 1) / 2, 0, 1) * 255)``
    in float32 (the inverse direction of ``u8_to_unit``).  NaN inputs are outside the contract."""
    if x.dim() != 4 or x.shape[1] != 3 or x.dtype != torch.float32 or not x.is_cuda:
        raise ValueError(f"image_to_u8: x must be a float32 CUDA (B, 3, H, W) tensor, got {x.dtype} {tuple(x.shape)} on {x.device}")
    B, _, H, W = x.shape
    if out is None:
        out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=x.device)
    elif out.shape != (B, H, W, 3) or out.dtype != torch.uint8 or not out.is_contiguous():
        raise ValueError(f"image_to_u8: out must be a contiguous uint8 ({B}, {H}, {W}, 3) tensor")
    _lib.check(_lib.lib.gifb200_image_to_u8(x.data_ptr(), out.data_ptr(), B, H, W, *x.stride(), _lib.stream()), "image_to_u8")
    return out
