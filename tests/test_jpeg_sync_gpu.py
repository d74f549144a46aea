"""GPU: the device JPEG decoder gives Pillow's bits at every chunk size of its self-synchronising entropy decode -- from
16 B chunks, where nearly every segment is finished by the serial jpeg_sync_fix, to 1 MiB, where every segment is one
chunk -- on the corpus of tests/test_jpeg_sync_cpu.py (whose host restatement shows which regime each case takes), on the
project's own encoder's files, and it still reports corrupt files per image.  Fixtures are made here from seeded arrays."""
import io
import time
from functools import lru_cache

import numpy as np
import pytest
import torch
from PIL import Image

from gif_b200.synth_images import flat, jpeg, noise, photo
from test_jpeg_sync_cpu import BIG, CHUNKS, corpus, derived_chunks, truncated_with_restarts

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="no CUDA device")]

BIG_GPU_CHUNKS = (16, 128, 1024)


@lru_cache(maxsize=None)
def pil_rgb(b):
    return np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))


def decode(blobs, chunk_bytes):
    from gif_b200.image_decode import decode_jpeg_batch
    imgs, status = decode_jpeg_batch(list(blobs), chunk_bytes=chunk_bytes)
    return [im.cpu().numpy() for im in imgs], status.cpu().numpy()


def assert_pillow(names, blobs, imgs, status, chunk_bytes):
    bad = [n for n, s in zip(names, status) if s != 0]
    assert not bad, (chunk_bytes, bad[:5])
    for n, b, got in zip(names, blobs, imgs):
        ref = pil_rgb(b)
        assert got.shape == ref.shape and np.array_equal(got, ref), \
            (chunk_bytes, n, int((got != ref).sum()) if got.shape == ref.shape else got.shape)


def small():
    return [(n, b) for n, b in corpus() if f"{BIG}x{BIG}" not in n]


def big():
    return [(n, b) for n, b in corpus() if f"{BIG}x{BIG}" in n]


@pytest.mark.parametrize("chunk_bytes", CHUNKS)
def test_every_chunk_size_decodes_pillows_bits(chunk_bytes, capsys):
    """The whole corpus as one mixed batch, then every image on its own; the 1024² q100 4:2:0 images at 16, 128 and
    1024 B, timed."""
    cases = small() + (big() if chunk_bytes in BIG_GPU_CHUNKS else [])
    names, blobs = zip(*cases)
    assert_pillow(names, blobs, *decode(blobs, chunk_bytes), chunk_bytes)
    for n, b in cases:
        torch.cuda.synchronize()
        t = time.perf_counter()
        imgs, status = decode([b], chunk_bytes)
        if f"{BIG}x{BIG}" in n:
            with capsys.disabled():
                print(f"\n{n} at {chunk_bytes} B: {1e3 * (time.perf_counter() - t):.1f} ms (decode + copy back)")
        assert_pillow([n], [b], imgs, status, chunk_bytes)


def test_segment_end_on_and_past_a_chunk_boundary():
    """Per image, the chunk sizes that make the first segment exactly one chunk, end exactly on a chunk boundary of
    several, end one byte past one (a last chunk of padding only), and put every chunk start on an MCU start."""
    for n, b in corpus():
        for cb in derived_chunks(b):
            assert_pillow([n], [b], *decode([b], cb), cb)


def test_round_trip_through_the_device_encoder():
    """Files written by encode_jpeg_batch decode at 16 B and 1 KB to what Pillow decodes from the same bytes."""
    from gif_b200.image_encode import encode_jpeg_batch
    for (h, w) in ((256, 256), (72, 100), (1024, 1024)):
        x = np.stack([np.asarray(photo(h, w, 3)), np.asarray(noise(h, w, 4)), np.asarray(flat(h, w, 5))])
        for q in ((100,) if h == 1024 else (75, 100)):
            files = encode_jpeg_batch(torch.from_numpy(x).cuda(), quality=q)
            names = [f"{k}-{h}x{w}-q{q}" for k in ("photo", "noise", "flat")]
            for cb in (16, 1024):
                assert_pillow(names, files, *decode(files, cb), cb)


def missing_restart_interval():
    """A file with restart intervals from which one interval (and its marker) has been cut out."""
    data = jpeg(photo(64, 64, 13), quality=95, restart_marker_blocks=2)
    sos = data.index(b"\xff\xda")
    rst = [i for i in range(sos, len(data) - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]
    assert len(rst) > 3
    return data[:rst[1]] + data[rst[2]:]


@pytest.mark.parametrize("chunk_bytes", (16, 128, 1024))
def test_corruption_reported_per_image_at_every_chunk_size(chunk_bytes):
    """Corrupt scan bytes, a file cut in half, one cut inside its restart intervals and one missing an interval: each gets
    a nonzero status, and the good images between them still decode to Pillow's bits."""
    from gif_b200.image_decode import parse_jpeg
    good = [jpeg(photo(64, 64, s), quality=95) for s in range(4)] + [jpeg(noise(48, 80, 1), quality=100)]
    bad = bytearray(jpeg(photo(64, 64, 10), quality=95))
    sos = bad.index(b"\xff\xda") + 14
    rng = np.random.default_rng(0)
    bad[sos + 40:sos + 400] = bytes(rng.integers(0, 255, 360, dtype=np.uint8))     # no 0xFF: stays one segment
    full = jpeg(photo(64, 64, 11), quality=95)
    missing = missing_restart_interval()
    assert len(parse_jpeg(missing)["segments"][-1]) == 0
    blobs = [good[0], bytes(bad), good[1], full[:len(full) // 2], good[2], truncated_with_restarts(), good[3], missing, good[4]]
    imgs, status = decode(blobs, chunk_bytes)
    bad_idx = (1, 3, 5, 7)
    assert all(status[i] != 0 for i in bad_idx), status
    for i in range(0, len(blobs), 2):
        assert status[i] == 0 and np.array_equal(imgs[i], pil_rgb(blobs[i])), (chunk_bytes, i, status)


def test_chunk_bytes_outside_the_api_range_raise():
    from gif_b200._lib import GifB200Error
    b = jpeg(photo(32, 32, 1), quality=90)
    for cb in (15, (1 << 20) + 1):
        with pytest.raises(GifB200Error, match="chunk_bytes"):
            decode([b], cb)
    decode([b], 16)
    decode([b], 1 << 20)
