"""GPU: a corruption that only the device decoders detect -- a PNG scanline with filter type 5 (its chunk CRCs and zlib
stream valid) and a JPEG whose entropy-coded bytes are scrambled -- is reported, naming the image, by every caller of the
shared decode path: ``prepare_multiscale_lmdb`` (which also leaves no output behind), ``real_image_statistics`` and
``DeviceBatchLoader`` (for a real-image key, a render key and a normal-map key)."""
import os

import numpy as np
import pytest
import torch

from gif_b200.image_decode import UnsupportedImage, host_decode
from gif_b200.synth_images import build_lmdbs, jpeg, photo, png, png_chunks

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="no CUDA device")]


def bad_filter_png(size, seed):
    """An RGB PNG whose middle scanline has filter type 5."""
    rows = np.asarray(photo(size, size, seed)).reshape(size, size * 3)
    raw = np.concatenate([np.zeros((size, 1), np.uint8), rows], 1)
    raw[size // 2, 0] = 5
    return png_chunks(size, size, 2, raw.tobytes())


def scrambled_jpeg(seed):
    """A 64x64 JPEG with 360 entropy-coded bytes replaced by random ones (no 0xFF, so its markers stay intact)."""
    data = bytearray(jpeg(photo(64, 64, seed), quality=95))
    sos = data.index(b"\xff\xda") + 14
    data[sos + 40:sos + 400] = bytes(np.random.default_rng(0).integers(0, 255, 360, dtype=np.uint8))
    return bytes(data)


def test_the_corruptions_pass_the_host_checks():
    assert host_decode(bad_filter_png(40, 1), "p").kind == "png"
    assert host_decode(scrambled_jpeg(10), "j").kind == "jpeg"


@pytest.mark.parametrize("kind", ["png", "jpeg"])
def test_prepare_multiscale_lmdb_names_the_file(tmp_path, kind):
    from gif_b200.prepare_images import prepare_multiscale_lmdb
    src = tmp_path / "src" / "c"
    os.makedirs(src)
    for i in range(3):
        (src / f"{i}.png").write_bytes(png(photo(64, 64, i)))
    (src / f"bad.{kind}").write_bytes(bad_filter_png(64, 9) if kind == "png" else scrambled_jpeg(10))
    with pytest.raises(UnsupportedImage, match=f"bad.{kind}: "):
        prepare_multiscale_lmdb(tmp_path / "src", tmp_path / "out", sizes=(8, 16), batch_size=2)
    assert sorted(os.listdir(tmp_path)) == ["src"]


class _Features(torch.nn.Module):
    def forward(self, x):
        return [x]


def test_real_image_statistics_names_the_file(tmp_path):
    from gif_b200.fid_real import real_image_statistics
    for i in range(3):
        (tmp_path / f"{i}.png").write_bytes(png(photo(40, 40, i)))
    (tmp_path / "1_bad.png").write_bytes(bad_filter_png(40, 9))
    with pytest.raises(UnsupportedImage, match="1_bad.png: corrupt PNG scanlines"):
        real_image_statistics(tmp_path, 64, _Features(), 3)


@pytest.mark.parametrize("which", ["real", "render", "normal map"])
def test_device_batch_loader_names_the_key(tmp_path, which):
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset, LmdbReader, image_key, normal_map_key, write_lmdb
    lmdbs = dict(zip(("real", "rend"), build_lmdbs(tmp_path, 4, 64, 32)))
    db, key, bad = {"real": ("real", image_key(64, 2), scrambled_jpeg(10)),
                    "render": ("rend", image_key(32, 1), bad_filter_png(32, 9)),
                    "normal map": ("rend", normal_map_key(32, 3), bad_filter_png(32, 8))}[which]
    r = LmdbReader(lmdbs[db])
    items = dict(r.items())
    r.close()
    items[key] = bad
    lmdbs[db] = str(tmp_path / "corrupt")
    write_lmdb(lmdbs[db], items.items())
    ds = GifLmdbDataset(lmdbs["real"], lmdbs["rend"], np.zeros((4, 3), np.float32), resolution=64, rend_flm_res=32)
    with pytest.raises(UnsupportedImage, match=f"^{key.decode()}: corrupt"):
        for _ in DeviceBatchLoader(ds, 4, shuffle=False):
            pass
