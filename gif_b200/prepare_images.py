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
    """Read and host-decode one file (``image_decode.host_decode``: dispatched on its magic bytes as ``Image.open`` does):
    (the ``HostImage``, its comment).  Anything the device decoders cannot read raises ``UnsupportedImage`` naming the file."""
    with open(path, "rb") as f:
        data = f.read()
    im = I.host_decode(data, path)
    return im, (_png_comment if im.kind == "png" else _jpeg_comment)(data)


def decoded_groups(loaded, device):
    """One batch of ``load_image`` results decoded on the device (Image.convert("RGB")) and grouped by shape
    (``image_decode.shape_groups``), so each group is resized in one call.  A corrupt image raises ``UnsupportedImage``
    naming its file."""
    batch = I.DecodeBatch([im for im, _ in loaded])
    images, status = batch.decode(device)
    I.check_status(status.cpu(), batch.names)
    return I.shape_groups(images)


def resized_crops(groups, n, size):
    """``decoded_groups`` of n images -> (n, size, size, 3): torchvision's resize(size, LANCZOS) + center_crop(size) of
    each, Pillow-exact."""
    out = None
    for idx, x in groups:
        (rw, rh), (left, top) = I.resized_crop_box(x.shape[2], x.shape[1], size)
        r = I.resize_lanczos_u8(x, (rh, rw))[:, top:top + size, left:left + size]
        if idx == list(range(n)):                  # one group, the whole batch in input order
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
                for k, loaded in enumerate(I.prefetch(pool, load_image, batches)):
                    groups = decoded_groups(loaded, device)
                    comments = [c for _, c in loaded]
                    first = k * batch_size
                    for s in sizes:
                        blobs = encode_jpeg_batch(resized_crops(groups, len(loaded), s), quality, comments)
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
