"""numpy restatement of the device JPEG encoder (gif_b200/csrc/jpeg_encode.cu), stage by stage, written from JPEG (ITU-T
T.81) and the libjpeg conventions Pillow's output shows.  tests/test_prepare_images_cpu.py pins its bytes to Pillow's
``save(format="JPEG", quality=q)``; the kernels restate these functions.  The headers and tables are the host code's
(gif_b200/image_encode.py); everything from the pixels to the stuffed entropy-coded bytes is here."""
import numpy as np

from gif_b200 import image_encode as E
from gif_b200.image_decode import _NATURAL

SCALEBITS = 16
ONE_HALF = 1 << (SCALEBITS - 1)


def _fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


def rgb_to_ycc(rgb):
    """libjpeg's rgb_ycc_convert in 16-bit fixed point; Cb / Cr round with 0.5 - epsilon so they never reach 256."""
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    y = (_fix(0.29900) * r + _fix(0.58700) * g + _fix(0.11400) * b + ONE_HALF) >> SCALEBITS
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + (128 << SCALEBITS) + ONE_HALF - 1) >> SCALEBITS
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + (128 << SCALEBITS) + ONE_HALF - 1) >> SCALEBITS
    return y, cb, cr


def component_planes(rgb):
    """uint8 (H, W, 3) -> (Y, Cb, Cr) sample planes padded to whole MCUs: Y (16*my, 16*mx), chroma (8*my, 8*mx).

    Luma is replicated from the last column / row.  Chroma is h2v2-downsampled from full-resolution planes whose right edge
    is replicated to 16*mx columns and whose odd last row is doubled; each output is (a + b + c + d + bias) >> 2 with the
    bias alternating 1, 2 along the row; rows past the image's chroma height repeat the last downsampled row."""
    H, W, _ = rgb.shape
    mx, my, _ = E.block_layout(W, H)
    y, cb, cr = rgb_to_ycc(rgb)
    rows = np.minimum(np.arange(16 * my), H - 1)
    cols = np.minimum(np.arange(16 * mx), W - 1)
    Y = y[rows][:, cols]
    ch = (H + 1) // 2
    crow = np.minimum(np.arange(8 * my), ch - 1)
    r0, r1 = np.minimum(2 * crow, H - 1), np.minimum(2 * crow + 1, H - 1)
    c0, c1 = np.minimum(2 * np.arange(8 * mx), W - 1), np.minimum(2 * np.arange(8 * mx) + 1, W - 1)
    bias = np.where(np.arange(8 * mx) % 2 == 0, 1, 2)
    out = [Y]
    for p in (cb, cr):
        out.append((p[r0][:, c0] + p[r0][:, c1] + p[r1][:, c0] + p[r1][:, c1] + bias) >> 2)
    return out


C = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069,
         c2053=16819, c2562=20995, c3072=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, first):
    """One pass of libjpeg's islow (Loeffler-Ligtenberg-Moschytz) FDCT along axis -1 (13-bit constants, 2 extra bits of
    precision kept after the first pass)."""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = np.empty_like(d)
    sh = 13 - 2 if first else 13 + 2
    o[..., 0] = (t10 + t11) << 2 if first else _descale(t10 + t11, 2)
    o[..., 4] = (t10 - t11) << 2 if first else _descale(t10 - t11, 2)
    z1 = (t12 + t13) * C["c0541"]
    o[..., 2] = _descale(z1 + t13 * C["c0765"], sh)
    o[..., 6] = _descale(z1 - t12 * C["c1847"], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * C["c1175"]
    t4, t5, t6, t7 = t4 * C["c0298"], t5 * C["c2053"], t6 * C["c3072"], t7 * C["c1501"]
    z1, z2, z3, z4 = -z1 * C["c0899"], -z2 * C["c2562"], -z3 * C["c1961"] + z5, -z4 * C["c0390"] + z5
    o[..., 7] = _descale(t4 + z1 + z3, sh)
    o[..., 5] = _descale(t5 + z2 + z4, sh)
    o[..., 3] = _descale(t6 + z2 + z3, sh)
    o[..., 1] = _descale(t7 + z1 + z4, sh)
    return o


def fdct_islow(blocks):
    """int (..., 8, 8) samples -> FDCT coefficients scaled by 8 (natural order), samples centred on 128 first."""
    d = blocks.astype(np.int64) - 128
    d = _fdct_1d(d, True)
    return np.swapaxes(_fdct_1d(np.swapaxes(d, -1, -2), False), -1, -2)


def quantise(coef, table):
    """libjpeg-turbo's reciprocal quantisation of natural-order coefficients with one table: zigzag int (..., 64)."""
    zz = coef.reshape(*coef.shape[:-2], 64)[..., _NATURAL]
    rcs = np.array([E.reciprocal(8 * int(v)) for v in table[_NATURAL]], np.int64)
    a = np.abs(zz)
    q = ((a + rcs[:, 1]) * rcs[:, 0]) >> (16 + rcs[:, 2])
    return np.where(zz < 0, -q, q)


def _blocks(plane):
    h, w = plane.shape
    return plane.reshape(h // 8, 8, w // 8, 8).swapaxes(1, 2)       # (by, bx, 8, 8)


def scan_blocks(rgb, quality):
    """Quantised zigzag blocks in scan order (MCU by MCU: Y00 Y01 Y10 Y11 Cb Cr) with the component of each: int (n, 64),
    int (n,).  Luma blocks wholly outside the image (the MCU grid overhangs it) are dummy blocks: zero AC, and the DC of the
    block before them in the MCU -- the left neighbour at the right edge, the MCU's top-right block at the bottom."""
    H, W, _ = rgb.shape
    mx, my, n = E.block_layout(W, H)
    qt = E.quant_tables(quality)
    Y, Cb, Cr = component_planes(rgb)
    qy = quantise(fdct_islow(_blocks(Y)), qt[0])                     # (2my, 2mx, 64)
    qb, qr = (quantise(fdct_islow(_blocks(p)), qt[1]) for p in (Cb, Cr))
    wb, hb = -(-W // 8), -(-H // 8)
    out = np.zeros((my, mx, 6, 64), np.int64)
    for j in range(4):
        dy, dx = j >> 1, j & 1
        out[:, :, j] = qy[dy::2, dx::2]
    out[:, :, 4], out[:, :, 5] = qb, qr
    if wb % 2:                                                       # right dummy column in the last MCU column
        for j in (1, 3):
            out[:, -1, j] = 0
            out[:, -1, j, 0] = out[:, -1, j - 1, 0]
    if hb % 2:                                                       # bottom dummy row in the last MCU row
        for j in (2, 3):
            out[-1, :, j] = 0
            out[-1, :, j, 0] = out[-1, :, 1, 0]
    return out.reshape(n, 64), np.tile([0, 0, 0, 0, 1, 2], mx * my)


def _nbits(v):
    return int(abs(int(v))).bit_length()


def block_codes(blk, last_dc, dc_tab, ac_tab):
    """Huffman codes of one block as (code, length) pairs: DC difference, then AC run/size symbols (ZRL for 16 zeros, EOB
    after the last nonzero coefficient unless it is the 64th); each magnitude follows its code in ``nbits`` bits, negative
    values as v - 1 in two's complement."""
    out = []
    diff = int(blk[0]) - last_dc
    s = _nbits(diff)
    out.append((dc_tab[s] & 0xFFFF, dc_tab[s] >> 16))
    if s:
        out.append(((diff - 1 if diff < 0 else diff) & ((1 << s) - 1), s))
    run = 0
    for k in range(1, 64):
        v = int(blk[k])
        if v == 0:
            run += 1
            continue
        while run > 15:
            out.append((ac_tab[0xF0] & 0xFFFF, ac_tab[0xF0] >> 16))
            run -= 16
        s = _nbits(v)
        sym = run << 4 | s
        out.append((ac_tab[sym] & 0xFFFF, ac_tab[sym] >> 16))
        out.append(((v - 1 if v < 0 else v) & ((1 << s) - 1), s))
        run = 0
    if run:
        out.append((ac_tab[0] & 0xFFFF, ac_tab[0] >> 16))
    return out


def entropy_bits(blocks, comps):
    """Per-block code lengths and the concatenated bit string (a list of 0/1) of the scan; DC differences chain per
    component in scan order from 0."""
    tabs = [E.huffman_codes(*t) for t in E.STD_HUFFMAN]
    last = [0, 0, 0]
    lengths, bits = [], []
    for blk, c in zip(blocks, comps):
        t = 0 if c == 0 else 2
        codes = block_codes(blk, last[c], tabs[t], tabs[t + 1])
        last[c] = int(blk[0])
        lengths.append(sum(n for _, n in codes))
        for code, n in codes:
            bits += [(code >> (n - 1 - i)) & 1 for i in range(n)]
    return np.array(lengths), bits


def pack_and_stuff(bits):
    """Bit string -> bytes: padded to a whole byte with 1-bits, every 0xFF byte followed by a stuffed 0x00."""
    bits = bits + [1] * (-len(bits) % 8)
    raw = np.packbits(np.array(bits, np.uint8)).tobytes() if bits else b""
    return raw.replace(b"\xff", b"\xff\x00")


def encode(rgb, quality=100, comment=None):
    """uint8 (H, W, 3) -> the JPEG file Pillow writes for ``Image.fromarray(rgb).save(f, "JPEG", quality=quality)``."""
    H, W, _ = rgb.shape
    blocks, comps = scan_blocks(rgb, quality)
    _, bits = entropy_bits(blocks, comps)
    return E.jpeg_file(W, H, quality, pack_and_stuff(bits), comment)
