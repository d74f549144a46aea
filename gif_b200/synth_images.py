"""Seeded synthetic images and LMDBs in the reference's on-disk format, for the image-decoder tests and
tools/bench_input.py: photo-like (1/f spectrum), noise and flat images, encoded with Pillow or (PNG) by hand."""
import io
import os
import struct
import zlib

import numpy as np
from PIL import Image


def photo(h, w, seed=0, mode="RGB"):
    """Seeded image with a photo-like (1/f) spectrum."""
    rng = np.random.default_rng(seed)
    c = {"RGB": 3, "RGBA": 4, "L": 1}[mode]
    f = np.fft.fftfreq(h)[:, None] ** 2 + np.fft.fftfreq(w)[None, :] ** 2
    out = []
    for _ in range(c):
        spec = (rng.standard_normal((h, w)) + 1j * rng.standard_normal((h, w))) / np.maximum(f, 1e-4) ** 0.75
        x = np.real(np.fft.ifft2(spec))
        out.append((x - x.min()) / (np.ptp(x) + 1e-9) * 255)
    a = np.clip(np.stack(out, -1), 0, 255).astype(np.uint8)
    return Image.fromarray(a[..., 0] if c == 1 else a, mode)


def jpeg(img, **kw):
    b = io.BytesIO()
    img.save(b, "JPEG", **kw)
    return b.getvalue()


def png(img, **kw):
    b = io.BytesIO()
    img.save(b, "PNG", **kw)
    return b.getvalue()


def png_chunks(w, h, ct, raw, depth=8, interlace=0, idat_parts=1):
    def chunk(t, body):
        return struct.pack(">I", len(body)) + t + body + struct.pack(">I", zlib.crc32(body, zlib.crc32(t)))
    z = zlib.compress(raw)
    step = -(-len(z) // idat_parts)
    return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ct, 0, 0, interlace)) + \
        b"".join(chunk(b"IDAT", z[i:i + step]) for i in range(0, len(z), step)) + chunk(b"IEND", b"")


def noise(h, w, seed, mode="RGB"):
    rng = np.random.default_rng(seed)
    shape = (h, w) if mode == "L" else (h, w, {"RGB": 3, "RGBA": 4}[mode])
    return Image.fromarray(rng.integers(0, 256, shape, dtype=np.uint8), mode)


def flat(h, w, seed):
    a = np.zeros((h, w, 3), np.uint8)
    a[:] = np.random.default_rng(seed).integers(0, 256, 3, dtype=np.uint8)
    a[h // 2:, : w // 3] = 17
    return Image.fromarray(a)


def png_folder(root, n, size, seed=0):
    """``n`` photo-like RGB PNGs of size x size written by Pillow as ``root/{i:05d}.png`` (FFHQ's naming); returns the paths."""
    os.makedirs(root, exist_ok=True)
    paths = []
    for i in range(n):
        paths.append(os.path.join(str(root), f"{i:05d}.png"))
        photo(size, size, seed + i).save(paths[-1], "PNG")
    return paths


def build_lmdbs(root, n, R, rr):
    """Real and render LMDBs as the reference's writers build them: LANCZOS resize + centre crop + JPEG q100, PNG renders."""
    from gif_b200.data import image_key, normal_map_key, write_lmdb
    real, rend = [(b"length", str(n).encode())], []
    for i in range(n):
        src = photo(R + 37, R + 11, 100 + i).resize((R + 20, R + 6), Image.LANCZOS)
        left, top = (src.size[0] - R) // 2, (src.size[1] - R) // 2
        real.append((image_key(R, i), jpeg(src.crop((left, top, left + R, top + R)), quality=100)))
        rend.append((image_key(rr, i), png(photo(rr, rr, 500 + i))))
        rend.append((normal_map_key(rr, i), png(noise(rr, rr, 900 + i) if i % 2 else photo(rr, rr, 700 + i))))
    write_lmdb(os.path.join(str(root), "real"), real)
    write_lmdb(os.path.join(str(root), "rend"), rend)
    return os.path.join(str(root), "real"), os.path.join(str(root), "rend")
