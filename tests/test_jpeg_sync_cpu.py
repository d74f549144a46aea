"""CPU: the self-synchronising entropy decode of the device JPEG decoder (csrc/image_decode.cu, DESIGN §5), restated on the
host by oracle/jpeg_sync_oracle.py, ends in the in-order decode's state at every chunk boundary for every corpus image and
chunk size; the corpus provably drives every regime of the schedule (consistent after init, after each sweep, finished by
jpeg_sync_fix) and its edge cases; and mutations of the schedule are caught.  The corpus is shared with
tests/test_jpeg_sync_gpu.py, which decodes it on the device at the same chunk sizes."""
from collections import Counter
from functools import lru_cache

import numpy as np
import pytest

from gif_b200 import image_decode as I
from gif_b200.synth_images import flat, jpeg, noise, photo
from oracle import jpeg_sync_oracle as O

CONTENT = {"photo": lambda h, w, s, mode="RGB": photo(h, w, s, mode), "noise": noise, "flat": lambda h, w, s, mode=None: flat(h, w, s)}
SIZES = [(1, 1), (7, 9), (17, 33), (63, 65), (256, 256)]
CASES = [dict(quality=q, subsampling=s) for q in (50, 75, 100) for s in (0, 1, 2)] + [dict(quality=90, optimize=True)] + \
    [dict(quality=95, restart_marker_blocks=r) for r in (1, 2, 7, 64)]
BIG = 1024                                # q100 4:2:0 photo and noise: the training LMDB's format
CHUNKS = (16, 24, 100, 128, 512, 1024, 4093, 1 << 20)
BIG_CHUNKS = (16, 128, 512, 1024)
COUNT_CHUNKS = (16, 128, 512, 1024)


def _name(kind, h, w, kw):
    return f"{kind}-{h}x{w}-" + "-".join(f"{a}{b}" for a, b in kw.items())


@lru_cache(maxsize=1)
def corpus():
    """(name, JPEG bytes) of every corpus image, from seeded arrays: photo / noise / flat content at every size and case,
    greyscale photo and noise, and the 1024² q100 4:2:0 photo and noise images last."""
    out = []
    for h, w in SIZES:
        for kind, make in CONTENT.items():
            for i, kw in enumerate(CASES):
                out.append((_name(kind, h, w, kw), jpeg(make(h, w, 31 * h + w + i), **kw)))
        for kind in ("photo", "noise"):
            for q in (75, 100):
                out.append((_name(kind + "L", h, w, dict(quality=q)), jpeg(CONTENT[kind](h, w, h + q, "L"), quality=q)))
    for kind in ("photo", "noise"):
        out.append((_name(kind, BIG, BIG, dict(quality=100)), jpeg(CONTENT[kind](BIG, BIG, 9), quality=100)))
    return tuple(out)


def truncated_with_restarts():
    """A file cut inside its scan, with restart intervals: the missing intervals become empty segments."""
    full = jpeg(photo(64, 64, 12), quality=95, restart_marker_blocks=2)
    return full[:len(full) * 2 // 3]


@lru_cache(maxsize=None)
def segments(blob):
    return tuple(O.segments(I.JpegBatch([I.parse_jpeg(blob)])))


def derived_chunks(blob):
    """Chunk sizes that put the first segment's end exactly on a chunk boundary -- one chunk (its length), several (a
    divisor of its length) -- or one byte past one (its length - 1: the last chunk holds only padding), and one whose
    boundaries fall on MCU starts of the in-order decode, so every guessed start state is exact; all at least the API's
    16 bytes."""
    sg = segments(blob)[0]
    n = sg.nbytes
    out = {n, n - 1}
    out.update([d for d in range(16, n // 2 + 1) if n % d == 0][:1])
    tr = sg.truth()
    out.update([p >> 3 for p, b, k in zip(tr.pos, tr.blk, tr.k) if p % 8 == 0 and b == k == 0 and 16 <= p >> 3 < n][:1])
    return sorted(c for c in out if 16 <= c <= (1 << 20))


def chunk_sizes(name, blob):
    return (BIG_CHUNKS if name.startswith(("photo-1024", "noise-1024")) else CHUNKS) + tuple(derived_chunks(blob))


@lru_cache(maxsize=None)
def sched(blob, seg_index, chunk_bytes, **mut):
    return O.schedule(segments(blob)[seg_index], chunk_bytes, **mut)


def all_schedules():
    for name, blob in corpus():
        for cb in chunk_sizes(name, blob):
            for si, sg in enumerate(segments(blob)):
                yield name, cb, sg, sched(blob, si, cb)


def test_kernel_sweeps_read_from_source():
    assert O.kernel_sweeps() == 3


def test_chunking_matches_jpeg_batch():
    """The restatement cuts segments into the chunks JpegBatch gives the kernels."""
    blobs = [b for _, b in corpus()[::23]] + [truncated_with_restarts()]
    for cb in (16, 100, 1 << 20):
        jb = I.JpegBatch([I.parse_jpeg(b) for b in blobs], cb)
        rows = jb.ints[jb.int_offsets[1]:jb.int_offsets[2]].reshape(-1, I.SEG_INTS)
        assert [int(r[6]) for r in rows] == [O.n_chunks(int(r[2]), cb) for r in rows]


def test_step_function_restatements_agree():
    """Segment.run (per-position tables, following the in-order decode once it meets it) equals the symbol-at-a-time
    ``run`` from random states, ends and segments, including states in the padding and on invalid codes."""
    rng = np.random.default_rng(5)
    picks = [b for _, b in corpus()[1::17]] + [truncated_with_restarts()]
    for blob in picks:
        for sg in segments(blob)[:3]:
            if sg.nbits == 0:
                continue
            for _ in range(40):
                pos = int(rng.integers(0, sg.nbits))
                s = O.pack(pos, int(rng.integers(0, sg.bpm)), int(rng.choice([0, 0, 1, 2, 40, 63])))
                end = min(sg.nbits, pos + int(rng.integers(1, 4000)))
                if rng.random() < 0.2:
                    end = sg.nbits
                want = O.run(sg.data, sg.nbits, s, end, sg.tables, sg.desc)
                assert sg.run(s, end) == want and sg.run(s, end, use_truth=False) == want


def test_truth_decodes_every_block():
    """The in-order decode of every valid segment completes its MCUs' blocks and stops in the padding."""
    for name, blob in corpus():
        for sg in segments(blob):
            tr = sg.truth()
            assert tr.final != O.KINVALID and tr.nblk == sg.want_blocks, name
            assert sg.nbits - 8 < tr.end_pos <= sg.nbits, name


def test_schedule_matches_truth():
    """Init, the kernel's sweeps, check and fix end in the in-order decode's state at every chunk boundary, with every
    chunk's start state, and the chunks' blocks add up to the segment's."""
    n = 0
    for name, cb, sg, s in all_schedules():
        errs = O.check_against_truth(sg, s)
        assert not errs, (name, cb, s.regime, errs[:5])
        assert sum(s.nblk) == sg.want_blocks, (name, cb)
        n += 1
    assert n > 3000


# regime / fact -> the least number of (image, chunk size, segment) cases of the corpus that must show it
COVERAGE = {
    "init (several chunks)": 10, "sweep1": 20, "sweep2": 5, "sweep3": 3, "fix": 100,
    "fix breaks past its last inconsistent chunk": 10, "fix runs to the segment's end": 10,
    "a chunk finishes no block": 100, "a chunk sees an invalid predecessor in a sweep": 5,
    "last chunk is 1 byte": 20, "segment is exactly one chunk": 20, "segment shorter than a chunk": 100,
    "segment is empty": 1,
}


def coverage():
    got = Counter()
    for name, cb, sg, s in all_schedules():
        if s.regime == "init":
            got["init (several chunks)"] += s.n > 1
        else:
            got[s.regime] += 1
        if s.regime == "fix":
            got["fix breaks past its last inconsistent chunk"] += s.fix_exit == "break"
            got["fix runs to the segment's end"] += s.fix_exit == "end"
        got["a chunk finishes no block"] += any(s.zero_blocks)
        got["a chunk sees an invalid predecessor in a sweep"] += any(s.invalid_pred)
        got["last chunk is 1 byte"] += s.n > 1 and s.short_last
        got["segment is exactly one chunk"] += sg.nbytes == cb
        got["segment shorter than a chunk"] += sg.nbytes < cb
    p = I.parse_jpeg(truncated_with_restarts())
    assert p["truncated"]
    for sg in segments(truncated_with_restarts()):
        if sg.nbytes == 0:
            s = O.schedule(sg, 16)
            assert s.n == 1 and s.nblk == [0] and s.out == [0] and s.regime == "init"
            got["segment is empty"] += 1
    return got


def test_every_regime_is_covered(capsys):
    got = coverage()
    with capsys.disabled():
        print("\njpeg sync corpus coverage (image, chunk size, segment cases): " + "; ".join(f"{k} {got[k]}" for k in COVERAGE))
    short = {k: (got[k], v) for k, v in COVERAGE.items() if got[k] < v}
    assert not short, short


def test_regime_counts(capsys):
    """One line: segments per regime at 16 / 128 / 512 / 1024 B on the 256² and 1024² photo and noise images (q100;
    the 256² ones 4:2:0 as well as the 1024² ones).  Counts of cases, not timings."""
    picks = [(n, b) for n, b in corpus() if n in ("photo-256x256-quality100-subsampling2", "noise-256x256-quality100-subsampling2",
                                                  "photo-1024x1024-quality100", "noise-1024x1024-quality100")]
    assert len(picks) == 4
    parts = []
    for cb in COUNT_CHUNKS:
        c = Counter()
        for name, blob in picks:
            for si in range(len(segments(blob))):
                s = sched(blob, si, cb)
                c[s.regime] += 1
        parts.append(f"{cb} B: " + " ".join(f"{r} {c[r]}" for r in O.REGIMES))
    with capsys.disabled():
        print("\njpeg sync regimes (256² + 1024² photo, noise; q100 4:2:0): " + "; ".join(parts))


MUTATIONS = [dict(skip_fix=True), dict(fix_stops_at_hi=True), dict(stale_sweep_nblk=True)]


@pytest.mark.parametrize("mut", MUTATIONS, ids=lambda m: next(iter(m)))
def test_mutations_break_truth(mut):
    """Each mutation of the schedule makes the truth comparison fail somewhere on the corpus: the corpus tells a
    correct schedule from a wrong one."""
    caught = 0
    for name, blob in corpus():
        for cb in chunk_sizes(name, blob):
            for si, sg in enumerate(segments(blob)):
                if sched(blob, si, cb).regime == "init" and "stale_sweep_nblk" not in mut:
                    continue
                s = sched(blob, si, cb, **mut)
                caught += bool(O.check_against_truth(sg, s))
        if caught >= 5:
            break
    assert caught >= 5, mut


def test_without_sweeps_the_fix_alone_is_exact():
    """With 0 sweeps the chain is still exact -- jpeg_sync_fix finishes any segment on its own -- but every segment that
    init left inconsistent goes to the serial fix: the sweeps only keep it rare."""
    more = 0
    for name, blob in corpus()[::3]:
        for cb in (16, 128, 1024):
            for si, sg in enumerate(segments(blob)):
                s = sched(blob, si, cb, sweeps=0)
                assert not O.check_against_truth(sg, s), (name, cb)
                assert s.regime in ("init", "fix")
                more += s.regime == "fix" and sched(blob, si, cb).regime != "fix"
    assert more > 20
