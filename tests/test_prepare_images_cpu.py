"""CPU: the pieces of the multiscale image LMDB writer that need no device -- Pillow's Lanczos coefficients (through a
numpy two-pass resample), the resize + centre-crop geometry, the JPEG encoder's numpy oracle byte for byte against
Pillow, the ImageFolder file order, and the streaming LMDB writer."""
import hashlib
import io
import os
import random

import numpy as np
import pytest
from PIL import Image

from gif_b200 import image_decode as I
from gif_b200 import image_encode as E
from gif_b200.data import LmdbReader, LmdbWriter, write_lmdb
from gif_b200.prepare_images import IMG_EXTENSIONS, _jpeg_comment, _png_comment, image_files
from gif_b200.synth_images import flat, noise, photo, png
from oracle import jpeg_encode_oracle as O


# ---------------------------------------------------------------------------------------------------------------- resize
def resample(a, coeffs, axis):
    """Pillow's 8bpc resample pass along ``axis`` of a uint8 (H, W, 3) array with a coefficient table, in float64 (every
    product and sum is an integer below 2^53, so the arithmetic is exact)."""
    n_in = a.shape[axis]
    dense = np.zeros((coeffs.shape[0], n_in))
    for r, row in enumerate(coeffs):
        dense[r, row[0]:row[0] + row[1]] = row[2:2 + row[1]]
    x = np.moveaxis(a, axis, 0).astype(np.float64)
    y = np.tensordot(dense, x, axes=(1, 0)) + (1 << 21)
    y = np.clip(np.floor(y / (1 << 22)), 0, 255).astype(np.uint8)
    return np.moveaxis(y, 0, axis)


def lanczos_numpy(a, w, h):
    if a.shape[1] != w:
        a = resample(a, I.lanczos_coeffs(a.shape[1], w), 1)
    if a.shape[0] != h:
        a = resample(a, I.lanczos_coeffs(a.shape[0], h), 0)
    return a


RESIZE_CASES = [((1024, 1024), (s, s)) for s in (8, 16, 32, 64, 128, 256, 512)] + [
    ((20, 20), (57, 57)), ((8, 8), (1024, 1024)), ((37, 23), (16, 40)), ((300, 171), (128, 224)),   # up, mixed, non-square
    ((64, 48), (64, 20)), ((64, 48), (13, 48)), ((5, 5), (5, 5))]                                   # one axis / none kept


@pytest.fixture(scope="module")
def big_photo():
    return photo(1024, 1024, 11)


@pytest.mark.parametrize("src,dst", RESIZE_CASES, ids=lambda s: "x".join(map(str, s)))
def test_lanczos_matches_pillow(src, dst, big_photo):
    (h, w), (ho, wo) = src, dst
    img = big_photo if (h, w) == (1024, 1024) else photo(h, w, h * w)
    a = np.asarray(img)
    assert np.array_equal(lanczos_numpy(a, wo, ho), np.asarray(img.resize((wo, ho), Image.LANCZOS)))


def test_lanczos_coeffs_large_reduction():
    c = I.lanczos_coeffs(1024, 8)
    assert c.shape[1] - 2 == 769                   # ceil(3 * 128) * 2 + 1 taps
    assert (np.abs(c[:, 2:].sum(1) - (1 << 22)) <= 769).all()


def test_bicubic_coeffs_unchanged():
    """The shared restatement gives the bicubic tables it gave before Lanczos joined it (sha256 of the tables)."""
    h = hashlib.sha256()
    for i, o in [(16, 32), (256, 512), (256, 1024), (48, 32), (1024, 256), (7, 3)]:
        h.update(np.ascontiguousarray(I.bicubic_coeffs(i, o)).tobytes())
    assert h.hexdigest() == "c406cd85c81316abf36886265902c780d721288bf764d6c7196a8e9b8185f151"


def torchvision_geometry(w, h, size):
    """torchvision's resize(img, size) + center_crop(size) of a w x h PIL image: (resized size, crop offset), the offset
    read back from a crop of an image of pixel indices."""
    tv = pytest.importorskip("torchvision.transforms.functional")
    rw, rh = tv.resize(Image.new("L", (w, h)), size, Image.NEAREST).size
    idx = Image.fromarray(np.arange(rw * rh, dtype=np.int32).reshape(rh, rw))
    first = int(np.asarray(tv.center_crop(idx, size))[0, 0])
    return (rw, rh), (first % rw, first // rw)


GEOMETRY = [(1024, 1024, 8), (1000, 700, 256), (700, 1000, 256), (33, 20, 8), (20, 33, 16), (101, 100, 8), (100, 101, 64),
            (17, 9, 4), (9, 17, 4), (1024, 1023, 512), (5, 3, 2)]


@pytest.mark.parametrize("w,h,size", GEOMETRY)
def test_resized_crop_box_matches_torchvision(w, h, size):
    assert I.resized_crop_box(w, h, size) == torchvision_geometry(w, h, size)


def test_resized_crop_box_rules():
    # long side int(size * long / short); offsets rounded half to even, as Python's round
    assert I.resized_crop_box(33, 20, 8) == ((13, 8), (2, 0))          # (13 - 8) / 2 = 2.5 -> 2
    assert I.resized_crop_box(20, 35, 8) == ((8, 14), (0, 3))          # (14 - 8) / 2 = 3
    assert I.resized_crop_box(8, 15, 4) == ((4, 7), (0, 2))            # 1.5 -> 2
    assert I.resized_crop_box(1024, 1024, 256) == ((256, 256), (0, 0))


# ----------------------------------------------------------------------------------------------------------------- JPEG
def pillow_jpeg(a, quality, comment=None):
    im = Image.fromarray(a)
    if comment is not None:
        im.info["comment"] = comment
    b = io.BytesIO()
    im.save(b, format="jpeg", quality=quality)
    return b.getvalue()


ENC_SIZES = [(1, 1), (7, 7), (8, 8), (9, 9), (15, 15), (16, 16), (17, 17), (20, 33), (256, 256)]
CONTENT = {"noise": noise, "flat": flat, "photo": photo}


def content(kind, h, w):
    return np.asarray(CONTENT[kind](h, w, h * 31 + w))


@pytest.mark.parametrize("quality", [100, 95, 75, 50])
@pytest.mark.parametrize("kind", list(CONTENT))
@pytest.mark.parametrize("size", ENC_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_oracle_encoder_matches_pillow(size, kind, quality):
    a = content(kind, *size)
    assert O.encode(a, quality) == pillow_jpeg(a, quality)


@pytest.mark.parametrize("comment", [b"made by hand", "café (a PNG text chunk gives a str)", b"\xff\xd8 binary \x00"])
@pytest.mark.parametrize("size", [(1, 1), (17, 17), (20, 33)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_oracle_encoder_comment_matches_pillow(size, comment):
    a = content("photo", *size)
    assert O.encode(a, 100, comment) == pillow_jpeg(a, 100, comment)
    with pytest.raises(ValueError, match="65533"):
        E.comment_segment(b"x" * 65534)


def test_oracle_stages():
    """Stage checks the whole-file comparison cannot localise: tables, the dummy-block rule, stuffing."""
    for q in (100, 95, 75, 50, 10, 1):
        ref = pillow_jpeg(np.zeros((8, 8, 3), np.uint8), q)
        head, tail = E.jpeg_header(8, 8, q)
        assert ref.startswith(head + tail)
    assert all((t == 1).all() for t in E.quant_tables(100))
    # 1x1: three dummy luma blocks carry the real block's DC, so their DC differences are 0
    blocks, comps = O.scan_blocks(np.full((1, 1, 3), 200, np.uint8), 100)
    assert blocks.shape == (6, 64) and (blocks[:4, 0] == blocks[0, 0]).all() and not blocks[1:4, 1:].any()
    assert O.pack_and_stuff([1] * 8 + [0] * 3) == b"\xff\x00\x1f"


def test_source_comments():
    im = photo(9, 9, 1)
    b = io.BytesIO()
    from PIL import PngImagePlugin
    info = PngImagePlugin.PngInfo()
    info.add_text("comment", "hello é")
    im.save(b, "PNG", pnginfo=info)
    data = b.getvalue()
    assert _png_comment(data) == Image.open(io.BytesIO(data)).info["comment"]
    info = PngImagePlugin.PngInfo()
    info.add_itxt("comment", "zé", zip=True)
    b = io.BytesIO()
    im.save(b, "PNG", pnginfo=info)
    assert _png_comment(b.getvalue()) == Image.open(io.BytesIO(b.getvalue())).info["comment"]
    assert _png_comment(png(im)) is None
    j = pillow_jpeg(np.asarray(im), 90, b"a jpeg comment")
    assert _jpeg_comment(j) == Image.open(io.BytesIO(j)).info["comment"] == b"a jpeg comment"


# ---------------------------------------------------------------------------------------------------------- file order
def make_tree(root):
    names = ["b/x/2.PNG", "b/x/10.png", "b/.hidden.jpg", "b/readme.txt", "b/y.JpEg", "a/z/deep/1.png", "a/0.webp",
             "a/notes.md", "a/A.png", "a/a.png", "c d/img.tiff", "a/z/0.bmp"]
    for n in names:
        p = os.path.join(root, n)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        open(p, "wb").close()
    open(os.path.join(root, "top.png"), "wb").close()                 # not in a class directory: not an image of the set
    return names


def test_image_files_order(tmp_path):
    make_tree(tmp_path)
    got = [os.path.relpath(p, tmp_path) for p in image_files(tmp_path)]
    assert got == ["a/0.webp", "a/A.png", "a/a.png", "a/z/0.bmp", "a/z/deep/1.png", "b/.hidden.jpg", "b/x/10.png",
                   "b/x/2.PNG", "b/y.JpEg", "c d/img.tiff"]


def test_image_files_matches_imagefolder(tmp_path):
    datasets = pytest.importorskip("torchvision.datasets")
    from torchvision.datasets.folder import IMG_EXTENSIONS as TV_EXT
    assert tuple(TV_EXT) == IMG_EXTENSIONS
    make_tree(tmp_path)
    ref = [p for p, _ in sorted(datasets.ImageFolder(str(tmp_path), loader=lambda p: p).imgs, key=lambda x: x[0])]
    assert image_files(tmp_path) == ref


def test_image_files_errors(tmp_path):
    open(os.path.join(tmp_path, "loose.png"), "wb").close()
    with pytest.raises(FileNotFoundError, match="class folder"):
        image_files(tmp_path)
    os.makedirs(os.path.join(tmp_path, "empty"))
    with pytest.raises(FileNotFoundError, match="no valid file"):
        image_files(tmp_path)


# -------------------------------------------------------------------------------------------------------------- LMDB
def test_streaming_writer_round_trip_out_of_order(tmp_path):
    rng = random.Random(3)
    items = {f"{s}-{i:05d}".encode(): bytes(rng.randrange(256) for _ in range(rng.choice([0, 5, 1000, 2040, 2100, 9000, 70000])))
             for s in (8, 1024) for i in range(120)}
    items[b"length"] = b"120"
    keys = list(items)
    rng.shuffle(keys)
    with LmdbWriter(tmp_path / "db") as w:
        for k in keys:
            w.put(k, items[k])
    r = LmdbReader(str(tmp_path / "db"))
    assert len(r) == len(items)
    assert dict(r.items()) == items
    assert [k for k, _ in r.items()] == sorted(items)
    assert all(r.get(k) == v for k, v in items.items())
    r.close()
    with pytest.raises(ValueError, match="duplicate"):
        w = LmdbWriter(tmp_path / "dup")
        w.put(b"a", b"1")
        w.put(b"a", b"2")
        w.close()


def test_write_lmdb_bytes_unchanged(tmp_path):
    """``write_lmdb`` writes through the streaming writer the same data.mdb as before it (sha256 of the old writer's files)."""
    rng = random.Random(0)
    cases = {"small": [(b"k%03d" % i, bytes([i]) * (i * 7)) for i in range(50)],
             "mixed": [(f"{i:05d}".encode(), bytes(rng.randrange(256) for _ in range(rng.choice([3, 100, 2100, 5000, 20000]))))
                       for i in range(300)],
             "empty": [], "one": [(b"length", b"7")]}
    want = {"small": "9f70311c89719397f1ca52c3a955f288caaba87dfb868be043dde5eb207aa551",
            "mixed": "6663d6efa887e2b42fbdf0e66855f913c2c3caee0488386028e73edb80712f73",
            "empty": "0e075cc571f2529fbc2ae70556e64769324d3a998ce6630cf948f5cf3398be39",
            "one": "36cc0b9fe9441282dd5082f5a453e02095e1b7e46c23e6f4e55d8f5a9fba79ea"}
    for name, items in cases.items():
        p = write_lmdb(str(tmp_path / name), items)
        assert hashlib.sha256(open(p, "rb").read()).hexdigest() == want[name], name
