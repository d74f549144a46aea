"""FID statistics of the real images, computed on the device from a folder of PNGs: what the reference's
``FidComputer.compute_true_img_response`` does when its cache file is missing (my_utils/compute_fid.py:26-46, then
``fid_score.calculate_activation_statistics`` -> ``get_activations``, my_utils/pytorch_fid/fid_score.py:57-123, 199-221):

  1. the folder's ``*.png`` files, the first 50 000;
  2. whole batches of 32 only (the remainder is dropped), or one batch of all the files when there are fewer than 32;
  3. each image opened with Pillow and, only when the resolution R is not 299, ``resize((R, R))`` (bicubic; a plain copy
     when the image is already R x R); then ``/ 255`` in float32;
  4. the FID Inception features (its own bilinear resize to 299 and 2x - 1), then ``np.mean`` / ``np.cov`` in float64.

Here a host thread pool reads, parses and inflates the PNGs of batch k+1 (zlib releases the GIL) while the device undoes
the scanline filters (``image_decode.DecodeBatch``), resizes (``gifb200_resize_bicubic_u8``, bit-exact with Pillow) and
runs the network on batch k.  The native ``InceptionV3`` takes the uint8 batch as it is (``gifb200_resize_bilinear_u8`` reads
v / 255 inside its input resize); any other model gets the float batch v / 255.  ``fid.ActivationStatistics`` reduces the
features as they come.

One deliberate deviation: the reference takes ``glob``'s order, which is the directory order of the file system, so with
more than 50 000 files (FFHQ has 70 000) which images are used depends on the disk.  Here the names are sorted, so the
statistics are a function of the folder's contents.

Only 8-bit RGB PNGs are accepted, as in the reference, where a grey or palette image gives a 2-D array and RGBA four
channels, and either breaks the batch or the network.  Anything else raises ``UnsupportedImage`` naming the file."""
import collections
import glob
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import image_decode as I
from .fid import ActivationStatistics, compute_activation_batch

MAX_IMAGES = 50_000          # compute_fid.py:42
BATCH_SIZE = 32              # compute_fid.py:43
INCEPTION_SIZE = 299         # fid_score.py:104: no resize at this resolution


def real_image_files(root, limit=MAX_IMAGES, batch_size=BATCH_SIZE):
    """The files the statistics use: ``root/*.png`` (glob's case-sensitive match, no hidden files) in sorted order, the first
    ``limit``, cut to a whole number of batches -- or all of them when there are fewer than ``batch_size``."""
    files = sorted(glob.glob(os.path.join(glob.escape(os.fspath(root)), "*.png")))[:limit]
    if not files:
        raise FileNotFoundError(f"{root}: no *.png images to compute the real images' FID statistics from")
    if len(files) < batch_size:
        return files
    return files[:len(files) // batch_size * batch_size]


def load_png(path):
    """Read, parse and inflate one PNG on the host (``image_decode.host_decode``): ((W, H, 3, b""), inflated scanlines).
    8-bit RGB only."""
    with open(path, "rb") as f:
        im = I.host_decode(f.read(), path)
    if im.kind != "png" or im.bpp != 3:
        what = "JPEG" if im.kind == "jpeg" else ("grey" if im.bpp == 1 else "RGBA") + " PNG"
        raise I.UnsupportedImage(f"{path}: {what}: the FID statistics take 8-bit RGB PNGs only")
    return (im.w, im.h, im.bpp, b""), im.data


def device_batch(files, loaded, resolution, status, device):
    """One batch of ``load_png`` results on the device (``image_decode.DecodeBatch``) as the network's input: uint8
    (B, h, w, 3), the scanlines unfiltered and, where the reference resizes (R != 299 and the image is not already R x R),
    Pillow's bicubic resize to R x R; a batch of one shape that needs no resize is returned as a view.  ``status``: int32
    (B,) device words, zeroed by the caller, that receive the decode's status (``image_decode.check_status``)."""
    hdrs = [h for h, _ in loaded]
    if resolution == INCEPTION_SIZE:
        for f, (w, h, _, _) in zip(files, hdrs):
            if (w, h) != hdrs[0][:2]:
                raise ValueError(f"{f}: {w}x{h} in a batch of {hdrs[0][0]}x{hdrs[0][1]} images; at resolution 299 the images "
                                 "are not resized, so they must all have one size (the reference's np.array of the batch)")
    batch = I.DecodeBatch([I.HostImage(f, "png", w, h, bpp, raw) for f, ((w, h, bpp, _), raw) in zip(files, loaded)])
    groups = I.shape_groups(batch.decode(device, status)[0])

    def fit(x):
        keep = resolution == INCEPTION_SIZE or x.shape[1:3] == (resolution, resolution)
        return x if keep else I.resize_bicubic_u8(x, resolution)
    if len(groups) == 1:
        return fit(groups[0][1])
    out = torch.empty(len(files), resolution, resolution, 3, dtype=torch.uint8, device=device)
    for idx, x in groups:
        out[idx] = fit(x)
    return out


def real_image_statistics(root, resolution, model, dims, batch_size=BATCH_SIZE, threads=None, device=None,
                          limit=MAX_IMAGES):
    """(mu, sigma) float64 CUDA tensors of ``model``'s ``dims`` features over the real images in ``root`` at ``resolution``
    (see the module docstring).  ``threads``: host threads reading and inflating (default: the CPU count, at most 32)."""
    device = torch.device(device or "cuda")
    if device.type != "cuda":
        raise RuntimeError("the real images' FID statistics decode the PNGs on the device: they need a CUDA device")
    from .inception import InceptionV3
    native = isinstance(model, InceptionV3)
    files = real_image_files(root, limit, batch_size)
    bs = min(batch_size, len(files))
    batches = [files[i:i + bs] for i in range(0, len(files), bs)]
    status = torch.zeros(len(files), dtype=torch.int32, device=device)
    stats = ActivationStatistics(dims, device)
    inflight = collections.deque()                 # at most two batches queued on the device ahead of the host
    pool = ThreadPoolExecutor(threads or min(32, os.cpu_count() or 1))
    try:
        with torch.no_grad():
            for k, loaded in enumerate(I.prefetch(pool, load_png, batches)):
                if len(inflight) == 2:
                    inflight.popleft().synchronize()
                x = device_batch(batches[k], loaded, resolution, status[k * bs:(k + 1) * bs], device)
                if not native:                     # v / 255 with a true division (a CUDA 0-dim divisor, not a scalar)
                    x = x.permute(0, 3, 1, 2).float().div_(torch.full((), 255.0, device=device))
                stats.update(compute_activation_batch(model, x))
                ev = torch.cuda.Event()
                ev.record()
                inflight.append(ev)
    finally:
        pool.shutdown(wait=True, cancel_futures=True)
    I.check_status(status.cpu(), files)
    return stats.finalize()


def save_statistics(path, mu, sigma):
    """Write ``mu`` / ``sigma`` (float64) as the reference's ``np.savez`` cache, atomically: a temporary file in the same
    directory renamed into place, so a reader never sees a partial file."""
    d = os.path.dirname(os.path.abspath(path))
    os.makedirs(d, exist_ok=True)
    tmp = f"{path}.tmp{os.getpid()}"
    try:
        with open(tmp, "xb") as f:
            np.savez(f, mu=np.asarray(mu, np.float64), sigma=np.asarray(sigma, np.float64))
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
