"""CPU: the host side of the device image decoders -- JPEG marker and PNG chunk parsing on Pillow-written files, the
rejection of everything outside the supported subset, Pillow's bicubic coefficient tables, and the shared batch path
(``host_decode``, ``DecodeBatch``'s packing, ``check_status``, shape grouping, ``prefetch``)."""
import struct
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

from gif_b200 import image_decode as I
from gif_b200.synth_images import jpeg, photo, png, png_chunks


JPEG_CASES = [dict(quality=q, subsampling=s) for q in (50, 75, 100) for s in (0, 1, 2)] + \
    [dict(quality=90, optimize=True), dict(quality=100, restart_marker_blocks=1), dict(quality=95, restart_marker_blocks=7)]
SIZES = [(1, 1), (7, 9), (17, 33), (256, 256)]


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("kw", JPEG_CASES, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
def test_parse_jpeg(size, kw):
    h, w = size
    p = I.parse_jpeg(jpeg(photo(h, w, 1), **kw))
    assert (p["w"], p["h"], p["ncomp"]) == (w, h, 3)
    hs, vs = {0: (1, 1), 1: (2, 1), 2: (2, 2)}[kw.get("subsampling", 2)]
    assert (p["hs"], p["vs"]) == (hs, vs)
    assert (p["mcux"], p["mcuy"]) == (-(-w // (8 * hs)), -(-h // (8 * vs)))
    assert len(p["blk"]) == hs * vs + 2
    n_mcu = p["mcux"] * p["mcuy"]
    assert len(p["segments"]) == -(-n_mcu // p["dri"]) and not p["truncated"]
    for seg in p["segments"]:
        assert len(seg) > 0
    if kw.get("quality") == 100:
        assert all((q == 1).all() for q in p["q"])
    # the packed batch is self-consistent
    jb = I.JpegBatch([p])
    assert jb.n_seg == len(p["segments"]) and jb.n_chunk >= jb.n_seg
    assert jb.n_blocks == sum(a * b for a, b in zip(p["bw"], p["bh"]))


def test_parse_jpeg_greyscale_and_unstuffing():
    data = jpeg(photo(40, 24, 2, "L"), quality=100)
    p = I.parse_jpeg(data)
    assert p["ncomp"] == 1 and (p["mcux"], p["mcuy"]) == (3, 5) and len(p["segments"]) == 1
    raw = data[data.index(b"\xff\xda"):]
    assert len(p["segments"][0]) == len(raw) - 10 - 2 - raw.count(b"\xff\x00")     # SOS (marker + 8), EOI


def test_huffman_table_standard_luma_dc():
    bits = (0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0)
    t = I.huffman_table(bits, tuple(range(12)))
    assert t[0b00 << 7] == (2 << 8) | 0            # code 00 -> symbol 0
    assert t[0b010 << 6] == (3 << 8) | 1
    assert t[0b111111110 << 0] == (9 << 8) | 11    # the longest code
    assert t[511] == 0                             # the reserved all-ones code
    with pytest.raises(I.UnsupportedImage, match="Huffman"):
        I.huffman_table((3,) + (0,) * 15, (0, 1, 2))
    with pytest.raises(I.UnsupportedImage, match="Huffman"):       # codes 0 and 1: the second is all ones, reserved
        I.huffman_table((2,) + (0,) * 15, (0, 1))


def test_rejects_unsupported_jpeg():
    img = photo(32, 32, 3)
    with pytest.raises(I.UnsupportedImage, match="progressive"):
        I.parse_jpeg(jpeg(img, progressive=True))
    with pytest.raises(I.UnsupportedImage, match="component"):
        I.parse_jpeg(jpeg(img.convert("CMYK")))
    data = jpeg(img)
    with pytest.raises(I.UnsupportedImage, match="truncated"):
        I.parse_jpeg(data[:300])
    with pytest.raises(I.UnsupportedImage, match="SOI"):
        I.parse_jpeg(b"GIF89a" + data)
    sof = data.index(b"\xff\xc0")
    with pytest.raises(I.UnsupportedImage, match="12-bit"):
        I.parse_jpeg(data[:sof + 4] + b"\x0c" + data[sof + 5:])
    with pytest.raises(I.UnsupportedImage, match="arithmetic"):
        I.parse_jpeg(data[:sof + 1] + b"\xc9" + data[sof + 2:])
    # marker segments whose length field is shorter than their contents
    with pytest.raises(I.UnsupportedImage, match="corrupt JPEG header"):
        I.parse_jpeg(data[:sof + 2] + b"\x00\x05" + data[sof + 4:])
    with pytest.raises(I.UnsupportedImage, match="corrupt JPEG header"):
        I.parse_jpeg(data[:sof] + b"\xff\xdd\x00\x02" + data[sof:])        # DRI without its interval


def test_parse_png_modes():
    for mode, bpp in (("RGB", 3), ("L", 1), ("RGBA", 4)):
        img = photo(19, 23, 4, mode)
        w, h, b, z = I.parse_png(png(img))
        assert (w, h, b) == (23, 19, bpp)
        assert len(I.inflate_png((w, h, b, z))) == h * (1 + w * bpp)


def test_rejects_unsupported_png():
    img = photo(16, 16, 5)
    with pytest.raises(I.UnsupportedImage, match="palette"):
        I.parse_png(png(img.convert("P")))
    with pytest.raises(I.UnsupportedImage, match="16-bit"):
        I.parse_png(png(Image.fromarray(np.arange(256, dtype=np.uint16).reshape(16, 16) * 200)))
    with pytest.raises(I.UnsupportedImage, match="interlaced"):
        I.parse_png(png_chunks(4, 4, 2, b"\0" * (4 * 13), interlace=1))
    data = bytearray(png(img))
    data[40] ^= 0x55
    with pytest.raises(I.UnsupportedImage, match="CRC"):
        I.parse_png(bytes(data))
    with pytest.raises(I.UnsupportedImage, match="truncated"):
        I.parse_png(png(img)[:-20])
    with pytest.raises(I.UnsupportedImage, match="corrupt PNG"):
        body = b"\x00" * 5
        I.parse_png(b"\x89PNG\r\n\x1a\n" + struct.pack(">I", 5) + b"IHDR" + body + struct.pack(">I", zlib.crc32(body, zlib.crc32(b"IHDR"))))
    with pytest.raises(I.UnsupportedImage, match="data stream"):
        I.inflate_png(I.parse_png(png_chunks(4, 4, 2, b"\0" * 20)))


def pillow_coeffs(in_size, out_size):
    """Pillow's own fixed-point weights, recovered from its output: resizing unit impulses of a 1-row image (horizontal
    pass only) gives, for each output sample, weight * 255 rounded -- enough to pin the tap ranges and signs."""
    rows = []
    for x in range(in_size):
        a = np.zeros((1, in_size), np.uint8)
        a[0, x] = 255
        rows.append(np.asarray(Image.fromarray(a).resize((out_size, 1), Image.BICUBIC), np.int32)[0])
    return np.stack(rows, 1)            # (out, in)


@pytest.mark.parametrize("sizes", [(16, 32), (256, 512), (256, 1024), (48, 32)])
def test_bicubic_coeffs(sizes):
    i, o = sizes
    c = I.bicubic_coeffs(i, o)
    ks = c.shape[1] - 2
    assert ks == int(np.ceil(2.0 * max(i / o, 1.0))) * 2 + 1
    assert (c[:, 0] >= 0).all() and (c[:, 0] + c[:, 1] <= i).all()
    # weights sum to one in 22-bit fixed point (up to the per-tap rounding)
    assert (np.abs(c[:, 2:].sum(1) - (1 << 22)) <= ks).all()
    # applied as Pillow applies them to 255-impulses they reproduce Pillow's output exactly
    dense = np.zeros((o, i), np.int64)
    for r in range(o):
        dense[r, c[r, 0]:c[r, 0] + c[r, 1]] = c[r, 2:2 + c[r, 1]]
    mine = np.clip(((255 * dense + (1 << 21)) >> 22), 0, 255)
    assert np.array_equal(mine, pillow_coeffs(i, o))


# ---------------------------------------------------------------------------------------------------------------- batches
def test_host_decode_dispatches_and_names_the_image():
    p = I.host_decode(png(photo(5, 7, 1, "RGBA")), "a.png")
    assert (p.name, p.kind, p.w, p.h, p.bpp, len(p.data)) == ("a.png", "png", 7, 5, 4, 5 * (1 + 7 * 4))
    j = I.host_decode(jpeg(photo(9, 11, 2)), "k-00001")
    assert (j.kind, j.w, j.h, j.bpp) == ("jpeg", 11, 9, 3) and j.data["segments"]
    bad = bytearray(png(photo(16, 16, 5)))
    bad[40] ^= 0x55
    for blob, msg in ((b"GIF89a" + bytes(20), "not a PNG or baseline JPEG"), (bytes(bad), "CRC"),
                      (jpeg(photo(32, 32, 3), progressive=True), "progressive")):
        with pytest.raises(I.UnsupportedImage, match=f"^img/x.bin: .*{msg}"):
            I.host_decode(blob, "img/x.bin")


def test_decode_batch_packs_a_mixed_batch_in_one_arena():
    imgs = [I.host_decode(png(photo(5, 7, 1)), "p0"), I.host_decode(jpeg(photo(9, 11, 2)), "j0"),
            I.host_decode(png(photo(3, 4, 3, "L")), "p1"), I.host_decode(jpeg(photo(17, 33, 4), quality=100), "j1")]
    b = I.DecodeBatch(imgs)
    assert b.order == [1, 3, 0, 2] and b.names == ["j0", "j1", "p0", "p1"]
    jb, pb = b.jpeg, b.png
    assert (jb.n_img, pb.n_img) == (2, 2) and b.out_bytes == jb.out_bytes + pb.out_bytes == b.png_out + pb.out_bytes
    # views in input order: the JPEGs at their JpegBatch offsets, then the PNGs after them
    assert b.views == [(jb.out_bytes + pb.out_offsets[0], 5, 7), (jb.out_offsets[0], 9, 11),
                       (jb.out_bytes + pb.out_offsets[1], 3, 4), (jb.out_offsets[1], 17, 33)]
    a, o = b.arena.numpy(), b.offsets
    assert (np.diff(o) % 256 == 0).all() and len(o) == 5
    assert a[o[0]:o[0] + len(jb.data)].tobytes() == jb.data
    assert a[o[1]:o[1] + pb.data_bytes].tobytes() == imgs[0].data + imgs[2].data
    assert np.array_equal(a[o[2]:o[2] + jb.ints.nbytes].view(np.int32), jb.ints)
    assert np.array_equal(a[o[3]:o[3] + pb.desc.nbytes].view(np.int32), pb.desc.ravel())
    only_png = I.DecodeBatch(imgs[::2])
    assert only_png.jpeg is None and only_png.order == [0, 1] and only_png.png_out == 0


def test_check_status_names_the_first_bad_image():
    I.check_status(np.zeros(3, np.int32), ["a", "b", "c"])
    with pytest.raises(I.UnsupportedImage, match=r"^b: corrupt or truncated JPEG data \(device status 1\), and 1 more images$"):
        I.check_status(np.array([0, I.STATUS_BAD_CODE, 0, I.STATUS_PNG_FILTER]), ["a", "b", "c", "d"])
    with pytest.raises(I.UnsupportedImage, match=r"^c: corrupt PNG scanlines .*status 4\)$"):
        I.check_status(torch.tensor([0, 0, I.STATUS_PNG_FILTER], dtype=torch.int32), ["a", "b", "c"])


def test_shape_groups_view_when_back_to_back():
    """A group lying back to back in the output buffer is returned as a view of it; otherwise it is stacked in input
    order.  A batch laid out by kind (JPEGs first) with one shape is one group with the identity indices."""
    buf = torch.arange(4 * 2 * 3 * 3 + 2 * 5 * 5 * 3, dtype=torch.int64).to(torch.uint8)
    a = [buf[k * 18:(k + 1) * 18].view(2, 3, 3) for k in range(4)]
    b = [buf[72 + k * 75:72 + (k + 1) * 75].view(5, 5, 3) for k in range(2)]
    groups = I.shape_groups([a[0], b[0], a[1], a[2], b[1], a[3]])
    assert [idx for idx, _ in groups] == [[0, 2, 3, 5], [1, 4]]
    for (idx, x), src in zip(groups, (a, b)):
        assert x.data_ptr() == src[0].data_ptr() and torch.equal(x, torch.stack(src))       # views
    mixed = [a[2], a[0], a[3], a[1]]                                                         # input order != buffer order
    (idx, x), = I.shape_groups(mixed)
    assert idx == [0, 1, 2, 3] and torch.equal(x, torch.stack(mixed)) and x.data_ptr() != a[0].data_ptr()
    assert torch.equal(I.as_batch([a[0], a[2]]), torch.stack([a[0], a[2]]))                   # a gap: a copy


def test_prefetch_runs_the_next_batch_while_this_one_is_used():
    from concurrent.futures import ThreadPoolExecutor
    batches = [[1, 2], [3], [4, 5, 6]]
    submitted = []

    class Pool(ThreadPoolExecutor):
        def submit(self, fn, x):
            submitted.append(x)
            return super().submit(fn, x)
    with Pool(2) as pool:
        got = []
        for k, r in enumerate(I.prefetch(pool, lambda x: 10 * x, batches)):
            got.append(r)
            assert submitted == sum(batches[:k + 2], [])           # batch k+1 is on the pool while batch k is used
    assert got == [[10, 20], [30], [40, 50, 60]]
