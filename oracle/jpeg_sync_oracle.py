"""Host restatement of the device JPEG decoder's self-synchronising entropy decode (csrc/image_decode.cu, DESIGN §5).

``run`` restates the step function ``jpeg_run<false>`` of csrc/image_decode.cuh (``Segment.run`` is the same step on
per-position tables); ``truth`` decodes a whole segment in order; ``schedule`` restates the kernels' schedule -- ``jpeg_sync_init``, ``kSweeps`` ping-pong sweeps of
``jpeg_sync_step``, ``jpeg_sync_check`` and the serial ``jpeg_sync_fix`` -- and reports which regime each segment ends
in.  Every step of the device schedule is deterministic, so this predicts chunk by chunk what the device computes.

The host parse is shared, not restated: the descriptors, segment rows and Huffman tables come from
``gif_b200.image_decode.JpegBatch`` (``segments``).  Plain Python and numpy; nothing here touches the device."""
import bisect
import os
import re
from functools import lru_cache

import numpy as np

from gif_b200 import image_decode as I

KINVALID = (1 << 64) - 1                  # the decoding state after an invalid code
LOOK, HUFF_MAX, HUFF_OFF, HUFF_VALS = 9, 512, 530, 548
REGIMES = ("init", "sweep1", "sweep2", "sweep3", "fix")
_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gif_b200", "csrc", "image_decode.cu")


def kernel_sweeps():
    """``kSweeps`` as csrc/image_decode.cu defines it, so the restatement runs the sweeps the kernels run."""
    with open(_CU) as f:
        m = re.search(r"constexpr int kSweeps = (\d+);", f.read())
    assert m, "kSweeps not found in image_decode.cu"
    return int(m.group(1))


def pack(pos, blk, k):
    return (pos << 16) | (blk << 8) | k


def unpack(s):
    return s >> 16, (s >> 8) & 255, s & 255


def _peek32(seg, p):
    """32 bits of seg from bit p, big-endian; bytes past the end read as zero."""
    b = p >> 3
    w = 0
    for i in range(5):
        w = (w << 8) | (seg[b + i] if b + i < len(seg) else 0)
    return (w >> (8 - (p & 7))) & 0xFFFFFFFF


def _huff_decode(t, win):
    """(symbol, length) of the code at the top of win, (-1, 0) for a code no table entry matches."""
    e = int(t[win >> (32 - LOOK)])
    if e:
        return e & 255, e >> 8
    for ln in range(LOOK + 1, 17):
        code = win >> (32 - ln)
        if code <= t[HUFF_MAX + ln]:
            return int(t[HUFF_VALS + ((code + int(t[HUFF_OFF + ln])) & 255)]), ln
    return -1, 0


def _table(desc, blk, k):
    comp = 0 if desc[I.JD_NCOMP] == 1 else int(desc[I.JD_BLK0 + blk]) & 15
    return int(desc[I.JD_DCT0 + comp]) if k == 0 else 2 + int(desc[I.JD_ACT0 + comp])


def run(seg, nbits, state, end, tables, desc):
    """``jpeg_run<false>``: decode from ``state`` until the bit position reaches ``end``.  Returns (state at the first symbol
    boundary at or after ``end``, blocks completed); KINVALID after an invalid code more than 16 bits before the segment's
    end.  A symbol that would run past ``nbits`` ends the run.  ``tables`` is the image's (4, HUFF_INTS) Huffman tables,
    ``desc`` its descriptor row.  One symbol at a time, straight from the bytes: the reference for ``Segment.run``."""
    if state == KINVALID:
        return KINVALID, 0
    pos, blk, k = unpack(state)
    bpm = int(desc[I.JD_BPM])
    nblk = 0
    while pos < end:
        sym, ln = _huff_decode(tables[_table(desc, blk, k)], _peek32(seg, pos))
        if sym < 0:
            if nbits - pos >= 16:
                return KINVALID, nblk
            break
        extra = sym if k == 0 else sym & 15
        if pos + ln + extra > nbits:
            break
        pos += ln + extra
        if k == 0:
            k = 1
        elif sym & 15:
            k += (sym >> 4) + 1
        else:
            k = k + 16 if sym >> 4 == 15 else 64
        if k >= 64:
            k = 0
            nblk += 1
            blk = blk + 1 if blk + 1 < bpm else 0
    return pack(pos, blk, k), nblk


def _windows16(seg, nbits):
    """The top 16 bits of the 32-bit window at every bit position of the segment (bytes past the end read as zero)."""
    a = np.frombuffer(bytes(seg) + b"\0\0\0", np.uint8).astype(np.uint32)
    p = np.arange(nbits, dtype=np.uint32)
    b = p >> 3
    w24 = (a[b] << 16) | (a[b + 1] << 8) | a[b + 2]
    return ((w24 >> (8 - (p & 7))) & 0xFFFF).astype(np.uint16)


@lru_cache(maxsize=64)
def _step_tables(t, dc):
    """``_huff_decode`` of a table (its int32 bytes) on all 65536 16-bit windows -- no code is longer -- as two uint8
    tables: the bits the symbol takes (code + extra bits; 0 for an invalid code) and the step of k (1 for a DC symbol; for
    AC r + 1, 16 for ZRL, 64 for EOB, which ends the block as coefficient 64 does)."""
    t = np.frombuffer(t, np.int32)
    adv, dk = np.zeros(65536, np.uint8), np.zeros(65536, np.uint8)
    for w in range(65536):
        sym, ln = _huff_decode(t, w << 16)
        if sym >= 0:
            r, s = sym >> 4, sym & 15
            adv[w] = ln + (sym if dc else s)
            dk[w] = 1 if dc else (r + 1 if s else (16 if r == 15 else 64))
    return adv, dk


class Segment:
    """One entropy-coded segment of a JpegBatch with its image's descriptor and tables, plus, per Huffman table it uses,
    the decode at every bit position (``_step_tables`` gathered at ``_windows16``), so that ``run`` costs a few byte lookups per symbol."""

    def __init__(self, data, desc, tables, first_mcu, n_mcu, image):
        self.data, self.desc, self.tables = bytes(data), np.asarray(desc), np.asarray(tables)
        self.nbytes, self.nbits = len(self.data), 8 * len(self.data)
        self.bpm = int(desc[I.JD_BPM])
        self.want_blocks = n_mcu * self.bpm
        self.image = image
        self._fast = None
        self._truth = None

    def _tables_fast(self):
        if self._fast is None:
            win = _windows16(self.data, self.nbits)
            per_table = {}
            for blk in range(self.bpm):
                for k in (0, 1):
                    ti = _table(self.desc, blk, k)
                    if ti not in per_table:
                        adv, dk = _step_tables(self.tables[ti].tobytes(), ti < 2)
                        per_table[ti] = (adv[win].tobytes(), dk[win].tobytes())
            self._fast = ([per_table[_table(self.desc, b, 0)][0] for b in range(self.bpm)],
                          [per_table[_table(self.desc, b, 1)] for b in range(self.bpm)])
        return self._fast

    def run(self, state, end, use_truth=True):
        """``run`` on this segment.  With ``use_truth``, a run that reaches a block start of the in-order decode follows
        it (the rest of the run is then determined) instead of decoding again."""
        if state == KINVALID:
            return KINVALID, 0
        dca, aca = self._tables_fast()
        tr = self.truth() if use_truth else None
        nbits, bpm = self.nbits, self.bpm
        pos, blk, k = unpack(state)
        nblk = 0
        while pos < end:
            if k == 0:
                if tr is not None:            # looked up at block starts only: cheaper, and as exact
                    i = tr.at.get(pos)
                    if i is not None and tr.blk[i] == blk and tr.k[i] == 0:
                        return tr.follow(i, end, nblk)
                a = dca[blk][pos]
                if not a:
                    if nbits - pos >= 16:
                        return KINVALID, nblk
                    break
                if pos + a > nbits:
                    break
                pos += a
                k = 1
            else:
                adv, dk = aca[blk]
                a = adv[pos]
                if not a:
                    if nbits - pos >= 16:
                        return KINVALID, nblk
                    break
                if pos + a > nbits:
                    break
                k += dk[pos]
                pos += a
                if k >= 64:
                    k = 0
                    nblk += 1
                    blk = blk + 1 if blk + 1 < bpm else 0
        return pack(pos, blk, k), nblk

    def truth(self):
        """The in-order decode of the whole segment from state 0 (``Truth``)."""
        if self._truth is None:
            self._truth = Truth(self)
        return self._truth


class Truth:
    """The sequential decode of a segment from its exact first state: the state at every symbol boundary (``pos``, ``blk``,
    ``k``; ``at`` maps a position to its index), blocks completed before each boundary (``cum``), and how it ended
    (``final``: the state after the last symbol, KINVALID after an invalid code; ``nblk``: blocks in the segment)."""

    def __init__(self, sg):
        dca, aca = sg._tables_fast()
        nbits, bpm = sg.nbits, sg.bpm
        pos = blk = k = nblk = 0
        P, B, K, C = [], [], [], []
        final = None
        while pos < nbits:
            P.append(pos)
            B.append(blk)
            K.append(k)
            C.append(nblk)
            if k == 0:
                a, step = dca[blk][pos], 1
            else:
                adv, dk = aca[blk]
                a, step = adv[pos], dk[pos]
            if not a:
                if nbits - pos >= 16:
                    final = KINVALID
                break
            if pos + a > nbits:
                break
            pos += a
            k = 1 if k == 0 else k + step
            if k >= 64:
                k = 0
                nblk += 1
                blk = blk + 1 if blk + 1 < bpm else 0
        if final is None and (not P or P[-1] != pos):       # the end state at nbits: the last boundary
            P.append(pos)
            B.append(blk)
            K.append(k)
            C.append(nblk)
        self.pos, self.blk, self.k, self.cum = P, B, K, C
        self.final = final if final is not None else pack(pos, blk, k)
        self.nblk = nblk
        self.end_pos = pos
        self.at = {p: i for i, p in enumerate(P)}

    def state(self, i):
        return pack(self.pos[i], self.blk[i], self.k[i])

    def follow(self, i, end, nblk):
        """The rest of a run that is at boundary i, stopping at the first boundary at or after ``end``.  Past the last
        boundary the run meets what ended the in-order decode there: the segment's end, or an invalid code."""
        j = bisect.bisect_left(self.pos, end, i)
        if j < len(self.pos):
            return self.state(j), nblk + self.cum[j] - self.cum[i]
        return self.final, nblk + self.cum[-1] - self.cum[i]

    def state_at_or_after(self, bit):
        """The in-order decode's state at its first boundary at or after ``bit`` (its end state past the last one)."""
        j = bisect.bisect_left(self.pos, bit)
        return self.state(j) if j < len(self.pos) else self.final


def truth(sg):
    """The in-order decode of segment ``sg`` from state 0."""
    return sg.truth()


def segments(jb):
    """The segments of a ``JpegBatch`` as ``Segment`` objects, from its packed descriptors, segment rows and tables."""
    o = jb.int_offsets
    desc = jb.ints[o[0]:o[1]].reshape(-1, I.DESC_INTS)
    rows = jb.ints[o[1]:o[2]].reshape(-1, I.SEG_INTS)
    huff = jb.ints[o[4]:o[5]].reshape(-1, 4, I.HUFF_INTS)
    return [Segment(jb.data[r[1]:r[1] + r[2]], desc[r[0]], huff[r[0]], int(r[3]), int(r[4]), int(r[0])) for r in rows]


def n_chunks(nbytes, chunk_bytes):
    """Chunks of a segment of nbytes (JpegBatch: at least one, so an empty segment gets one)."""
    return max(1, -(-nbytes // chunk_bytes))


class Schedule:
    """The result of ``schedule``: per chunk the final start state ``inp``, end state ``out`` and blocks ``nblk``; the
    segment's ``regime`` (one of REGIMES: the chain is consistent after init, after sweep 1..3, or only after the fix);
    the fix's range (``lo``, ``hi``, -1 without a fix) and how the fix loop ended (``fix_exit``: "break" past ``hi``, or
    "end" at the segment's last chunk); per-chunk facts: ``zero_blocks`` (finished no block), ``mid_symbol`` (its true start
    lies inside a symbol), ``invalid_pred`` (saw a KINVALID predecessor in a sweep), ``short_last`` (the last chunk holds
    fewer than 16 bits)."""


def schedule(sg, chunk_bytes, sweeps=None, skip_fix=False, fix_stops_at_hi=False, stale_sweep_nblk=False):
    """``jpeg_sync_init``, ``sweeps`` sweeps (default: the kernel's kSweeps), ``jpeg_sync_check`` and ``jpeg_sync_fix`` on
    one segment, exactly as the kernels order them.  The flags are mutations that the tests show the truth comparison
    catches or tolerates: ``skip_fix`` (no fix), ``fix_stops_at_hi`` (the fix never runs past the last inconsistent chunk
    the check saw), ``stale_sweep_nblk`` (a sweep re-decodes a chunk but keeps its old block count)."""
    sweeps = kernel_sweeps() if sweeps is None else sweeps
    n = n_chunks(sg.nbytes, chunk_bytes)
    bits = 8 * chunk_bytes

    def guess(c):
        return pack(c * bits, 0, 0)

    def chunk_run(c, s):
        end = sg.nbits if c + 1 == n else (c + 1) * bits
        if s == KINVALID:                 # restart from the guess: an invalid guessed run must not poison later chunks
            s = guess(c)
        return sg.run(s, end)

    inp = [guess(c) for c in range(n)]
    out, nblk = [], []
    for c in range(n):
        o, b = chunk_run(c, inp[c])
        out.append(o)
        nblk.append(b)
    invalid_pred = [False] * n

    def consistent(o):
        return all(o[c - 1] == inp[c] for c in range(1, n))

    regime = "init" if consistent(out) else None
    src = out
    for i in range(sweeps):
        dst = list(src)
        for c in range(1, n):
            if src[c - 1] != inp[c]:
                if src[c - 1] == KINVALID:
                    invalid_pred[c] = True
                inp[c] = src[c - 1]
                dst[c], b = chunk_run(c, src[c - 1])
                if not stale_sweep_nblk:
                    nblk[c] = b
        src = dst
        if regime is None and consistent(src):
            regime = f"sweep{i + 1}"
    out = src
    bad = [c for c in range(1, n) if out[c - 1] != inp[c]]
    lo, hi = (bad[0], bad[-1]) if bad else (-1, -1)
    fix_exit = None
    if bad and not skip_fix:
        regime = "fix"
        fix_exit = "end"
        for c in range(lo, n):
            if fix_stops_at_hi and c > hi:
                break
            if out[c - 1] == inp[c]:
                if c > hi:
                    fix_exit = "break"
                    break
                continue
            inp[c] = out[c - 1]
            out[c], nblk[c] = chunk_run(c, out[c - 1])
    s = Schedule()
    s.n, s.chunk_bytes, s.inp, s.out, s.nblk = n, chunk_bytes, inp, out, nblk
    s.regime, s.lo, s.hi, s.fix_exit = regime or "fix", lo, hi, fix_exit
    s.zero_blocks = [b == 0 for b in nblk]
    s.mid_symbol = [inp[c] != KINVALID and (inp[c] >> 16) > c * bits for c in range(n)]
    s.invalid_pred = invalid_pred
    s.short_last = sg.nbytes - (n - 1) * chunk_bytes < 2 if sg.nbytes else False
    return s


def check_against_truth(sg, s):
    """Where a schedule's final chain differs from the in-order decode: a list of (chunk, what) pairs, empty when the
    start state of every chunk is the in-order decode's state at its first boundary at or after the chunk's first bit
    (its predecessor's end state, as the decode defines it), the last chunk ends in the decode's end state, and the
    chunks' blocks add up to the decode's."""
    tr = sg.truth()
    bits = 8 * s.chunk_bytes
    errs = []
    for c in range(s.n):
        want_in = 0 if c == 0 else tr.state_at_or_after(c * bits)
        if s.inp[c] != want_in:
            errs.append((c, "in"))
        want_out = tr.final if c + 1 == s.n else tr.state_at_or_after((c + 1) * bits)
        if s.out[c] != want_out:
            errs.append((c, "out"))
    if sum(s.nblk) != tr.nblk:
        errs.append((-1, f"blocks {sum(s.nblk)} != {tr.nblk}"))
    return errs
