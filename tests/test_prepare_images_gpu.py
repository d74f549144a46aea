"""GPU: the multiscale image LMDB on the device -- the Lanczos resize and the JPEG encoder are byte-exact with Pillow, and
``prepare_multiscale_lmdb`` writes what the reference's recipe (Pillow + torchvision) writes, deterministically, and
leaves nothing behind when an input is corrupt.  Fixtures are made here from seeded arrays with Pillow."""
import hashlib
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image, PngImagePlugin

from gif_b200.synth_images import flat, jpeg, noise, photo, png
from test_prepare_images_cpu import CONTENT, ENC_SIZES, RESIZE_CASES, content, pillow_jpeg

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="no CUDA device")]


@pytest.mark.parametrize("src,dst", RESIZE_CASES, ids=lambda s: "x".join(map(str, s)))
def test_resize_lanczos_matches_pillow(src, dst):
    from gif_b200.image_decode import resize_lanczos_u8
    (h, w), (ho, wo) = src, dst
    srcs = [photo(h, w, 3), noise(h, w, 4), flat(h, w, 5)]
    x = torch.from_numpy(np.stack([np.asarray(s) for s in srcs])).cuda()
    y = resize_lanczos_u8(x, (ho, wo)).cpu().numpy()
    for k, s in enumerate(srcs):
        assert np.array_equal(y[k], np.asarray(s.resize((wo, ho), Image.LANCZOS))), k


@pytest.mark.parametrize("quality", [100, 95, 75, 50])
@pytest.mark.parametrize("size", ENC_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_encode_matches_pillow(size, quality):
    from gif_b200.image_encode import encode_jpeg_batch
    a = np.stack([content(kind, *size) for kind in CONTENT])
    comments = [None, b"a comment", "a str comment"]
    got = encode_jpeg_batch(torch.from_numpy(a).cuda(), quality, comments)
    for k in range(len(a)):
        assert got[k] == pillow_jpeg(a[k], quality, comments[k]), k


def test_encode_1024_batch_matches_pillow():
    from gif_b200.image_encode import encode_jpeg_batch
    a = np.stack([np.asarray(photo(1024, 1024, 1)), np.asarray(noise(1024, 1024, 2)), np.asarray(flat(1024, 1024, 3)),
                  np.asarray(photo(1024, 1024, 4))])
    x = torch.from_numpy(a).cuda()
    got = encode_jpeg_batch(x)
    for k in range(len(a)):
        assert got[k] == pillow_jpeg(a[k], 100), k
    assert encode_jpeg_batch(x) == got                       # deterministic


def reference_recipe(path, sizes, quality=100):
    """prepare_ffhq_multiscale_dataset.py's resize_worker: Pillow + torchvision."""
    tv = pytest.importorskip("torchvision.transforms.functional")
    img = Image.open(path).convert("RGB")
    out = []
    for s in sizes:
        r = tv.center_crop(tv.resize(img, s, Image.LANCZOS), s)
        b = io.BytesIO()
        r.save(b, format="jpeg", quality=quality)
        out.append(b.getvalue())
    return out


def make_folder(root):
    """Class directories of RGB / grey / RGBA PNGs, a JPEG input, a PNG with a comment, non-square images."""
    files = {
        "faces/00000.png": png(photo(1024, 1024, 1)),
        "faces/00001.png": png(photo(300, 200, 2, "L")),
        "faces/00002.png": png(photo(200, 333, 3, "RGBA")),
        "faces/sub/00003.jpg": jpeg(photo(257, 255, 4), quality=90),
        "faces/00004.PNG": png(noise(97, 131, 5)),
        "more/a.png": None,
        "more/b.jpeg": jpeg(photo(512, 512, 7), quality=100, comment=b"jpeg comment"),
    }
    info = PngImagePlugin.PngInfo()
    info.add_text("comment", "png comment")
    files["more/a.png"] = png(photo(64, 100, 6), pnginfo=info)
    for n, data in files.items():
        p = os.path.join(root, n)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(data)
    with open(os.path.join(root, "more", "notes.txt"), "w") as f:
        f.write("not an image")


def test_prepare_multiscale_lmdb_end_to_end(tmp_path):
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset, LmdbReader, PinnedBatchLoader, image_key, write_lmdb
    from gif_b200.prepare_images import image_files, prepare_multiscale_lmdb
    src = tmp_path / "src"
    make_folder(src)
    sizes = (8, 16, 32, 64, 128, 256, 512, 1024)
    files = image_files(src)
    n = prepare_multiscale_lmdb(src, tmp_path / "a", sizes=sizes, batch_size=3)
    assert n == len(files) == 7
    r = LmdbReader(str(tmp_path / "a"))
    assert r.get(b"length") == b"7" and len(r) == 7 * len(sizes) + 1
    for i, f in enumerate(files):
        for s, ref in zip(sizes, reference_recipe(f, sizes)):
            assert r.get(image_key(s, i)) == ref, (f, s)
    r.close()
    prepare_multiscale_lmdb(src, tmp_path / "b", sizes=sizes, batch_size=3, threads=2)
    digest = [hashlib.sha256(open(tmp_path / d / "data.mdb", "rb").read()).hexdigest() for d in ("a", "b")]
    assert digest[0] == digest[1]
    assert sorted(os.listdir(tmp_path)) == ["a", "b", "src"]
    with pytest.raises(FileExistsError):
        prepare_multiscale_lmdb(src, tmp_path / "a")
    # the LMDB feeds the training input at 256: the device loader's batches equal the PIL loader's
    rend = [(image_key(256, i), png(photo(256, 256, 50 + i))) for i in range(7)]
    rend += [(b"norm_map_" + image_key(256, i), png(photo(256, 256, 80 + i))) for i in range(7)]
    write_lmdb(str(tmp_path / "rend"), rend)
    ds = GifLmdbDataset(str(tmp_path / "a"), str(tmp_path / "rend"), np.zeros((7, 3), np.float32), resolution=256,
                        rend_flm_res=256)
    count = 0
    for a, b in zip(PinnedBatchLoader(ds, 3, shuffle=False, pin=False), DeviceBatchLoader(ds, 3, shuffle=False)):
        assert a[0].shape == (3, 3, 256, 256)
        for x, y in zip(a, b):
            assert torch.equal(x, y.cpu())
        count += 1
    assert count == 2


def test_corrupt_png_raises_and_leaves_nothing(tmp_path):
    from gif_b200.image_decode import UnsupportedImage
    from gif_b200.prepare_images import prepare_multiscale_lmdb
    src = tmp_path / "src" / "c"
    os.makedirs(src)
    for i in range(3):
        (src / f"{i}.png").write_bytes(png(photo(40, 40, i)))
    data = bytearray(png(photo(40, 40, 9)))
    data[60] ^= 0x5A                                                  # inside IDAT: fails its CRC
    (src / "bad.png").write_bytes(bytes(data))
    with pytest.raises(UnsupportedImage, match="bad.png"):
        prepare_multiscale_lmdb(tmp_path / "src", tmp_path / "out", sizes=(8, 16), batch_size=2)
    assert sorted(os.listdir(tmp_path)) == ["src"]
