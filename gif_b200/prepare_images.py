"""The multiscale training-image LMDB, built on the device: what the reference's
``prepare_lmdb/prepare_ffhq_multiscale_dataset.py`` writes, byte for byte, without ``lmdb``, torchvision or a Pillow
process pool.

For each image of ``torchvision.datasets.ImageFolder(root)``, sorted by path and numbered from 0, the reference stores,
for every size s in (8, 16, ..., 1024), ``Image.open(f).convert("RGB")`` -> ``resize(img, s, LANCZOS)`` (the short side
becomes s) -> ``center_crop(s)`` -> ``save(format="jpeg", quality=100)`` under the key ``f"{s}-{i:05d}"``, and finally
``length`` = the image count.  Here:

  host threads   read, parse and inflate batch k+1 (PNG: zlib; JPEG: markers and tables)             image_decode.py
  device         decodes batch k (PNG unfilter / baseline JPEG), resizes every size from the decoded image (not
                 cascaded, so each is bit-exact with Pillow), crops, and encodes the JPEGs              image_encode.py
  writer thread  appends the values to the LMDB as they come                                            data.LmdbWriter

Values reach the LMDB in batch order, so its bytes are a function of the images, the sizes, the quality and the batch
size (not of the thread count or timing).  The LMDB is written to ``out.tmp<pid>`` and renamed into place at the end; on
any error nothing is left behind."""
import os
import queue
import shutil
import struct
import threading
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import image_decode as I
from .data import LmdbWriter, image_key
from .image_encode import encode_jpeg_batch

SIZES = (8, 16, 32, 64, 128, 256, 512, 1024)
# torchvision.datasets.folder.IMG_EXTENSIONS, matched case-insensitively
IMG_EXTENSIONS = (".jpg", ".jpeg", ".png", ".ppm", ".bmp", ".pgm", ".tif", ".tiff", ".webp")


def image_files(root):
    """The reference's file list: ``ImageFolder(root).imgs`` (class directories sorted; each walked with
    ``sorted(os.walk(..., followlinks=True))`` and sorted names; hidden files included) sorted by path."""
    root = os.path.expanduser(os.fspath(root))
    classes = sorted(e.name for e in os.scandir(root) if e.is_dir())
    if not classes:
        raise FileNotFoundError(f"Couldn't find any class folder in {root}.")
    files = []
    for c in classes:
        found = []
        for d, _, names in sorted(os.walk(os.path.join(root, c), followlinks=True)):
            found += [os.path.join(d, n) for n in sorted(names) if n.lower().endswith(IMG_EXTENSIONS)]
        if not found:
            raise FileNotFoundError(f"Found no valid file for the classes {c}. Supported extensions are: "
                                    f"{', '.join(IMG_EXTENSIONS)}")
        files += found
    return sorted(files)


def _png_comment(data):
    """``im.info["comment"]`` of a PNG as Pillow reads it: the last tEXt / zTXt / iTXt chunk with the keyword "comment"
    (a str), else None."""
    pos, out = 8, None
    while pos + 12 <= len(data):
        ln, typ = struct.unpack_from(">I4s", data, pos)
        body = data[pos + 8:pos + 8 + ln]
        pos += 12 + ln
        if typ not in (b"tEXt", b"zTXt", b"iTXt") or not body.startswith(b"comment\0"):
            continue
        v = body[8:]
        try:
            if typ == b"tEXt":
                out = v.decode("latin-1")
            elif typ == b"zTXt":
                out = zlib.decompress(v[1:]).decode("latin-1")
            else:
                flag, _, rest = v[0], v[1], v[2:]
                rest = rest.split(b"\0", 2)[2]                     # language tag, translated keyword
                out = (zlib.decompress(rest) if flag else rest).decode("utf-8")
        except (zlib.error, UnicodeDecodeError, IndexError):
            continue
    return out


def _jpeg_comment(data):
    """``im.info["comment"]`` of a JPEG as Pillow reads it: the last COM segment before the scan (bytes), else None."""
    pos, out = 2, None
    while pos + 4 <= len(data) and data[pos] == 0xFF:
        m, ln = data[pos + 1], (data[pos + 2] << 8) | data[pos + 3]
        if m == 0xDA:
            break
        if m == 0xFE:
            out = data[pos + 4:pos + 2 + ln]
        pos += 2 + ln
    return out


def load_image(path):
    """Read and host-decode one file, dispatched on its magic bytes as ``Image.open`` does: ("png", (header, inflated
    scanlines)) or ("jpeg", parsed markers), and its comment.  Anything else raises ``UnsupportedImage`` naming the file."""
    with open(path, "rb") as f:
        data = f.read()
    try:
        if data[:8] == I._PNG_SIG:
            hdr = I.parse_png(data)
            return "png", (hdr[:3] + (b"",), I.inflate_png(hdr)), _png_comment(data)
        if data[:3] == b"\xff\xd8\xff":
            return "jpeg", I.parse_jpeg(data), _jpeg_comment(data)
        raise I.UnsupportedImage("not a PNG or baseline JPEG file (the device decoders read only these)")
    except I.UnsupportedImage as e:
        raise I.UnsupportedImage(f"{path}: {e}") from None


def _upload(parts, device):
    """Byte strings -> one uint8 device tensor, staged in pinned memory so the copy runs at full speed without blocking (the
    host allocator keeps the staging buffer until the copy has run)."""
    host = torch.empty(max(1, sum(len(p) for p in parts)), dtype=torch.uint8, pin_memory=True)
    a, o = host.numpy(), 0
    for p in parts:
        a[o:o + len(p)] = np.frombuffer(p, np.uint8)
        o += len(p)
    return host.to(device, non_blocking=True)


def _decode(files, loaded, device):
    """One batch of ``load_image`` results -> list of uint8 (H, W, 3) device tensors (Image.convert("RGB"))."""
    out = [None] * len(files)
    for kind in ("png", "jpeg"):
        idx = [i for i, l in enumerate(loaded) if l[0] == kind]
        if not idx:
            continue
        if kind == "png":
            hdrs, raws = zip(*(loaded[i][1] for i in idx))
            pb = I.PngBatch(hdrs, raws)
            buf = torch.empty(pb.out_bytes, dtype=torch.uint8, device=device)
            status = torch.zeros(pb.n_img, dtype=torch.int32, device=device)
            pb.launch(_upload(raws, device), I._to_device(pb.desc, device), buf, status)
            shapes, offs = pb.shapes, pb.out_offsets
        else:
            jb = I.JpegBatch([loaded[i][1] for i in idx])
            buf = torch.empty(jb.out_bytes, dtype=torch.uint8, device=device)
            status = torch.zeros(jb.n_img, dtype=torch.int32, device=device)
            ws = torch.empty(jb.workspace_bytes, dtype=torch.uint8, device=device)
            jb.launch(_upload([jb.data, b"\0"], device), I._to_device(jb.ints, device), buf, status, ws)
            shapes, offs = jb.shapes, jb.out_offsets
        bad = torch.nonzero(status).flatten().tolist()
        if bad:
            raise I.UnsupportedImage(f"{files[idx[bad[0]]]}: corrupt {kind.upper()} data")
        for k, i in enumerate(idx):
            h, w = shapes[k]
            out[i] = buf[offs[k]:offs[k] + h * w * 3].view(h, w, 3)
    return out


def shape_groups(images):
    """Images of one batch grouped by shape: [(indices, uint8 (n, H, W, 3))], so each group is resized in one call."""
    shapes = sorted({tuple(x.shape[:2]) for x in images})
    groups = []
    for shp in shapes:
        idx = [i for i, x in enumerate(images) if tuple(x.shape[:2]) == shp]
        groups.append((idx, torch.stack([images[i] for i in idx])))
    return groups


def resized_crops(groups, n, size):
    """``shape_groups`` of n images -> (n, size, size, 3): torchvision's resize(size, LANCZOS) + center_crop(size) of each,
    Pillow-exact."""
    out = None
    for idx, x in groups:
        (rw, rh), (left, top) = I.resized_crop_box(x.shape[2], x.shape[1], size)
        r = I.resize_lanczos_u8(x, (rh, rw))[:, top:top + size, left:left + size]
        if len(groups) == 1:
            return r.contiguous()
        if out is None:
            out = torch.empty(n, size, size, 3, dtype=torch.uint8, device=x.device)
        out[idx] = r
    return out


def prepare_multiscale_lmdb(root, out, sizes=SIZES, quality=100, batch_size=32, threads=None, device=None):
    """Write the multiscale image LMDB of the image tree ``root`` (ImageFolder layout) to the directory ``out``; returns the
    number of images.  ``threads``: host threads reading and inflating (default: the CPU count, at most 32)."""
    device = torch.device(device or "cuda")
    if device.type != "cuda":
        raise RuntimeError("the multiscale image LMDB is decoded, resized and encoded on the device: it needs a CUDA device")
    out = os.fspath(out)
    if os.path.exists(out):
        raise FileExistsError(f"{out} exists; the LMDB is written to a new directory")
    files = image_files(root)
    batches = [files[i:i + batch_size] for i in range(0, len(files), batch_size)]
    tmp = f"{out.rstrip(os.sep)}.tmp{os.getpid()}"
    pool = ThreadPoolExecutor(threads or min(32, os.cpu_count() or 1))
    values = queue.Queue(maxsize=4 * len(sizes))
    writer_error = []

    def write(w):
        try:
            while True:
                item = values.get()
                if item is None:
                    return
                for k, v in item:
                    w.put(k, v)
        except BaseException as e:              # reported by the main thread
            writer_error.append(e)
            while values.get() is not None:
                pass

    try:
        with LmdbWriter(tmp) as w:
            th = threading.Thread(target=write, args=(w,), daemon=True)
            th.start()
            try:
                nxt = [pool.submit(load_image, f) for f in batches[0]]
                for k, names in enumerate(batches):
                    loaded = [p.result() for p in nxt]
                    if k + 1 < len(batches):
                        nxt = [pool.submit(load_image, f) for f in batches[k + 1]]
                    groups = shape_groups(_decode(names, loaded, device))
                    comments = [l[2] for l in loaded]
                    first = k * batch_size
                    for s in sizes:
                        blobs = encode_jpeg_batch(resized_crops(groups, len(names), s), quality, comments)
                        values.put([(image_key(s, first + i), b) for i, b in enumerate(blobs)])
                    if writer_error:
                        break
                values.put([(b"length", str(len(files)).encode("utf-8"))])
            finally:
                values.put(None)
                th.join()
            if writer_error:
                raise writer_error[0]
        os.replace(tmp, out)
    except BaseException:
        shutil.rmtree(tmp, ignore_errors=True)
        raise
    finally:
        pool.shutdown(wait=True, cancel_futures=True)
    return len(files)
