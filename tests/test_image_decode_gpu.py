"""GPU: the device image decoders are bit-exact with Pillow (JPEG, PNG, bicubic resize), report corrupt data per image,
are deterministic, and ``DeviceBatchLoader`` yields bitwise the batches of ``PinnedBatchLoader``.  Fixtures are made here
from seeded arrays with Pillow."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

from gif_b200.synth_images import build_lmdbs, flat, jpeg, noise, photo, png, png_chunks
from test_image_decode_cpu import JPEG_CASES, SIZES

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="no CUDA device")]


def pil_rgb(b):
    return np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))


def check_jpeg(blobs):
    from gif_b200.image_decode import decode_jpeg_batch
    imgs, status = decode_jpeg_batch(blobs)
    assert (status.cpu() == 0).all()
    for i, (b, im) in enumerate(zip(blobs, imgs)):
        ref = pil_rgb(b)
        got = im.cpu().numpy()
        assert got.shape == ref.shape, i
        assert np.array_equal(got, ref), (i, int((got != ref).sum()), int(np.abs(got.astype(int) - ref).max()))


@pytest.mark.parametrize("kw", JPEG_CASES, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
def test_jpeg_matches_pillow(kw):
    blobs = []
    for h, w in SIZES:
        blobs += [jpeg(photo(h, w, h + w), **kw), jpeg(noise(h, w, h * w), **kw), jpeg(flat(h, w, h), **kw)]
    check_jpeg(blobs)


def test_jpeg_greyscale_and_mixed_batch():
    blobs = [jpeg(photo(h, w, 7, "L"), quality=q) for (h, w) in SIZES for q in (60, 100)]
    blobs += [jpeg(noise(h, w, 3), quality=100, subsampling=s) for (h, w), s in zip([(33, 17), (256, 256), (64, 96)], (0, 1, 2))]
    blobs += [jpeg(photo(1024, 1024, 9), quality=100), jpeg(noise(100, 300, 4), quality=98, restart_marker_blocks=3)]
    check_jpeg(blobs)


def test_jpeg_corrupt_and_truncated_reported_per_image():
    from gif_b200.image_decode import decode_jpeg_batch
    good = [jpeg(photo(64, 64, s), quality=95) for s in range(3)]
    bad = bytearray(jpeg(photo(64, 64, 10), quality=95))
    sos = bad.index(b"\xff\xda") + 14
    rng = np.random.default_rng(0)
    bad[sos + 40:sos + 400] = bytes(rng.integers(0, 255, 360, dtype=np.uint8))     # no 0xFF: stays one segment
    full = jpeg(photo(64, 64, 11), quality=95)
    trunc = full[:len(full) // 2]
    imgs, status = decode_jpeg_batch([good[0], bytes(bad), good[1], trunc, good[2]])
    st = status.cpu().numpy()
    assert st[1] != 0 and st[3] != 0 and st[0] == st[2] == st[4] == 0, st
    for i, g in ((0, good[0]), (2, good[1]), (4, good[2])):
        assert np.array_equal(imgs[i].cpu().numpy(), pil_rgb(g))


def test_jpeg_deterministic():
    from gif_b200.image_decode import decode_jpeg_batch
    blobs = [jpeg(photo(512, 512, s), quality=100) for s in range(4)]
    a = torch.cat([x.flatten() for x in decode_jpeg_batch(blobs)[0]])
    b = torch.cat([x.flatten() for x in decode_jpeg_batch(blobs)[0]])
    assert torch.equal(a, b)


def forced_filter_png(a, f):
    """PNG whose every row uses filter type f (0..4), built with numpy + zlib."""
    h, w = a.shape[:2]
    c = 1 if a.ndim == 2 else a.shape[2]
    x = a.reshape(h, w * c).astype(np.int32)
    out = np.zeros((h, 1 + w * c), np.uint8)
    out[:, 0] = f
    for r in range(h):
        up = x[r - 1] if r else np.zeros(w * c, np.int32)
        left = np.concatenate([np.zeros(c, np.int32), x[r, :-c]])
        ul = np.concatenate([np.zeros(c, np.int32), up[:-c]])
        if f == 0:
            p = 0
        elif f == 1:
            p = left
        elif f == 2:
            p = up
        elif f == 3:
            p = (left + up) >> 1
        else:
            pa, pb, pc = np.abs(up - ul), np.abs(left - ul), np.abs(left + up - 2 * ul)
            p = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
        out[r, 1:] = (x[r] - p) & 255
    return png_chunks(w, h, {1: 0, 3: 2, 4: 6}[c], out.tobytes(), idat_parts=3)


def test_png_matches_pillow():
    from gif_b200.image_decode import decode_png_batch
    blobs = []
    for mode in ("RGB", "L", "RGBA"):
        for (h, w) in [(1, 1), (7, 9), (17, 33), (256, 256), (300, 1025)]:
            img = photo(h, w, h + w, mode) if h > 1 else noise(h, w, 1, mode)
            blobs.append(png(img))
            a = np.asarray(noise(h, w, h * w + 1, mode))
            blobs += [forced_filter_png(a, f) for f in range(5)]
    imgs, status = decode_png_batch(blobs)
    assert (status.cpu() == 0).all()
    for i, (b, im) in enumerate(zip(blobs, imgs)):
        assert np.array_equal(im.cpu().numpy(), pil_rgb(b)), i


@pytest.mark.parametrize("sizes", [(16, 32), (256, 512), (256, 1024), (48, 32)])
def test_resize_matches_pillow(sizes):
    from gif_b200.image_decode import resize_bicubic_u8
    i, o = sizes
    srcs = [photo(i, i, 3), noise(i, i, 4), flat(i, i, 5)]
    x = torch.from_numpy(np.stack([np.asarray(s) for s in srcs])).cuda()
    y = resize_bicubic_u8(x, o).cpu().numpy()
    for k, s in enumerate(srcs):
        assert np.array_equal(y[k], np.asarray(s.resize((o, o)))), k


@pytest.mark.parametrize("R,rr", [(256, 256), (512, 256)])
def test_loader_equals_pinned_loader(tmp_path, R, rr):
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset, PinnedBatchLoader
    n, bs = 10, 4
    real, rend = build_lmdbs(tmp_path, n, R, rr)
    params = np.random.default_rng(1).standard_normal((n, 7)).astype(np.float32)
    ds = GifLmdbDataset(real, rend, params, resolution=R, rend_flm_res=rr, flame_mean=0.25, flame_std=1.5)
    pin, dev = PinnedBatchLoader(ds, bs, seed=3, pin=False), DeviceBatchLoader(ds, bs, seed=3)
    for _epoch in range(2):
        count = 0
        for a, b in zip(pin, dev):
            for x, y in zip(a, b):
                assert y.is_cuda and torch.equal(x, y.cpu())
            count += 1
        assert count == n // bs


def test_loader_names_the_corrupt_key(tmp_path):
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset, image_key, write_lmdb
    from gif_b200.image_decode import UnsupportedImage
    real, rend = build_lmdbs(tmp_path, 4, 64, 64)
    good = jpeg(photo(64, 64, 1), quality=100)
    bad = good[:len(good) // 2]
    write_lmdb(str(tmp_path / "real2"), [(b"length", b"4")] + [(image_key(64, i), bad if i == 2 else good) for i in range(4)])
    ds = GifLmdbDataset(str(tmp_path / "real2"), rend, np.zeros((4, 3), np.float32), resolution=64, rend_flm_res=64)
    with pytest.raises(UnsupportedImage, match="64-00002"):
        for _ in DeviceBatchLoader(ds, 4, shuffle=False):
            pass
