"""Input side of the hot path (SURVEY 8f.3): the reference's on-disk format -> pinned host batches -> the trainer.

The reference keeps its training images and its pre-rendered FLAME conditions in two LMDB environments
(dataset_loaders.py:157-182) written by prepare_lmdb/prepare_ffhq_multiscale_dataset.py:56-61 and
prepare_lmdb/create_deca_rendered_lmdb.py:57-89:

    real images       key  f"{resolution}-{index:05d}"            value  encoded image bytes (PNG / JPEG), RGB
    rendered FLAME    key  f"{resolution}-{index:05d}"            value  encoded texture render
    normal maps       key  f"norm_map_{resolution}-{index:05d}"   value  encoded normal-map render
    "length"          ASCII decimal number of images

and ``FFHQ.__getitem__`` (dataset_loaders.py:236-330) decodes them with PIL, maps to [-1, 1] (``ToTensor`` + ``Normalize(0.5, 0.5)``,
dataset_loaders.py:128-137) and returns ``(img, [cat(render, normal)], [flame_label], index)``.

This module reads that format WITHOUT the ``lmdb`` package (absent from the image; a dependency of the reference, not a
vendored source): ``LmdbReader`` is a read-only walker of LMDB's published file format (data.mdb: two meta pages, a B+tree of
branch / leaf pages with 2-byte node offsets, overflow pages for values larger than half a page), restated from the format
description in lmdb's mdb.c / lmdb.h (MDB_page, MDB_node, MDB_meta, MDB_db).  ``LmdbWriter`` is a streaming bulk writer of the
same format (overflow values appended as they arrive; packed leaves -> branch levels -> meta pages at the end) and
``write_lmdb`` its sorted-input form for fixtures.  PARITY UNPINNED: no LMDB file and
no lmdb library exist here to check either against; reader and writer are tested against each other and against the
documented layout constants (tests/test_data_cpu.py).

``GifLmdbDataset`` mirrors the reference dataset's item contract for the configuration the flagship run uses (rendered FLAME +
normal maps as condition); ``PinnedBatchLoader`` assembles whole batches in pinned host memory on a background thread, which is
exactly what ``GifTrainer.train_iteration`` / bench.py's ``e2e`` leg consume."""
import io
import os
import queue
import struct
import threading

import numpy as np
import torch

# ---------------------------------------------------------------------------------------------- LMDB file format
PAGE_HDR = 16                      # MDB_page: pgno u64, pad u16, flags u16, (lower u16, upper u16) | overflow page count u32
P_BRANCH, P_LEAF, P_OVERFLOW, P_META = 0x01, 0x02, 0x04, 0x08
F_BIGDATA = 0x01                   # node flag: the value lives in overflow pages, the node holds their first page number
MDB_MAGIC, MDB_VERSION = 0xBEEFC0DE, 1
P_INVALID = 0xFFFFFFFFFFFFFFFF
NODE_HDR = 8                       # MDB_node: lo u16, hi u16, flags u16, ksize u16


class LmdbFormatError(IOError):
    pass


class LmdbReader:
    """Read-only view of an LMDB environment's main database (``path`` = the directory holding data.mdb, or the file itself
    when the environment was created with ``subdir=False``)."""

    def __init__(self, path):
        if os.path.isdir(path):
            path = os.path.join(path, "data.mdb")
        self.path = path
        self._f = open(path, "rb")
        self._buf = np.memmap(path, dtype=np.uint8, mode="r")
        head = bytes(self._buf[:PAGE_HDR + 16])
        if struct.unpack_from("<I", head, PAGE_HDR)[0] != MDB_MAGIC:
            raise LmdbFormatError(f"{path}: not an LMDB data file (bad magic)")
        metas = []
        # the page size is not stored as such: it is the distance between the two meta pages; md_pad of the FREE_DBI record
        # of meta page 0 holds it (mdb.c: mm_psize is an alias of mm_dbs[FREE_DBI].md_pad)
        self.page_size = struct.unpack_from("<I", bytes(self._buf[PAGE_HDR + 24:PAGE_HDR + 28]), 0)[0]
        if self.page_size < 512 or self.page_size & (self.page_size - 1):
            raise LmdbFormatError(f"{path}: implausible page size {self.page_size}")
        for pg in (0, 1):
            off = pg * self.page_size
            flags = struct.unpack_from("<H", bytes(self._buf[off + 10:off + 12]), 0)[0]
            m = bytes(self._buf[off + PAGE_HDR:off + PAGE_HDR + 136])
            magic, version = struct.unpack_from("<II", m, 0)
            if not (flags & P_META) or magic != MDB_MAGIC:
                continue
            if version != MDB_VERSION:
                raise LmdbFormatError(f"{path}: unsupported LMDB data version {version}")
            # mm_address u64, mm_mapsize u64, mm_dbs[2] (48 bytes each), mm_last_pg u64, mm_txnid u64
            main = struct.unpack_from("<IHHQQQQQ", m, 24 + 48)
            last_pg, txnid = struct.unpack_from("<QQ", m, 24 + 96)
            metas.append({"txnid": txnid, "depth": main[2], "entries": main[6], "root": main[7], "last_pg": last_pg})
        if not metas:
            raise LmdbFormatError(f"{path}: no valid meta page")
        self.meta = max(metas, key=lambda d: d["txnid"])

    def close(self):
        self._buf = None
        self._f.close()

    def __len__(self):
        return self.meta["entries"]

    def _page(self, pgno):
        off = pgno * self.page_size
        return memoryview(self._buf[off:off + self.page_size])

    def _nodes(self, page):
        flags, lower = struct.unpack_from("<HH", page, 10)
        n = (lower - PAGE_HDR) // 2
        return flags, struct.unpack_from(f"<{n}H", page, PAGE_HDR)

    @staticmethod
    def _node(page, off):
        lo, hi, nflags, ksize = struct.unpack_from("<HHHH", page, off)
        return lo, hi, nflags, bytes(page[off + NODE_HDR:off + NODE_HDR + ksize])

    def _value(self, page, off, lo, hi, nflags, ksize):
        size = lo | (hi << 16)
        start = off + NODE_HDR + ksize
        if nflags & F_BIGDATA:
            pgno = struct.unpack_from("<Q", page, start)[0]
            o = pgno * self.page_size
            ov_flags, = struct.unpack_from("<H", bytes(self._buf[o + 10:o + 12]), 0)
            if not ov_flags & P_OVERFLOW:
                raise LmdbFormatError(f"page {pgno} is not an overflow page")
            return bytes(self._buf[o + PAGE_HDR:o + PAGE_HDR + size])
        return bytes(page[start:start + size])

    def get(self, key, default=None):
        """The value stored under ``key`` (bytes), or ``default``.  Keys compare as byte strings (LMDB's default order)."""
        if isinstance(key, str):
            key = key.encode("utf-8")
        pgno = self.meta["root"]
        if pgno == P_INVALID:
            return default
        while True:
            page = self._page(pgno)
            flags, ptrs = self._nodes(page)
            if flags & P_BRANCH:
                # child i covers keys >= separator i (separator 0 is empty): the last separator <= key
                lo_i, hi_i = 0, len(ptrs) - 1
                while lo_i < hi_i:
                    mid = (lo_i + hi_i + 1) // 2
                    if self._node(page, ptrs[mid])[3] <= key:
                        lo_i = mid
                    else:
                        hi_i = mid - 1
                lo, hi, nflags, _ = self._node(page, ptrs[lo_i])
                pgno = lo | (hi << 16) | (nflags << 32)
            elif flags & P_LEAF:
                lo_i, hi_i = 0, len(ptrs) - 1
                while lo_i <= hi_i:
                    mid = (lo_i + hi_i) // 2
                    lo, hi, nflags, k = self._node(page, ptrs[mid])
                    if k == key:
                        return self._value(page, ptrs[mid], lo, hi, nflags, len(k))
                    if k < key:
                        lo_i = mid + 1
                    else:
                        hi_i = mid - 1
                return default
            else:
                raise LmdbFormatError(f"page {pgno}: unexpected flags {flags:#x}")

    def items(self):
        """All (key, value) pairs in key order."""
        def walk(pgno):
            page = self._page(pgno)
            flags, ptrs = self._nodes(page)
            for off in ptrs:
                lo, hi, nflags, k = self._node(page, off)
                if flags & P_BRANCH:
                    yield from walk(lo | (hi << 16) | (nflags << 32))
                else:
                    yield k, self._value(page, off, lo, hi, nflags, len(k))
        if self.meta["root"] != P_INVALID:
            yield from walk(self.meta["root"])


class LmdbWriter:
    """Streaming bulk writer of an LMDB environment directory ``path`` (data.mdb) in the layout ``LmdbReader`` and readers
    of the published format expect: packed leaves, branch levels built bottom-up, values that do not fit half a page in
    overflow pages.  Values may arrive in any order (LMDB pages have no sibling links): ``put`` appends a large value's
    overflow pages to the file at once and keeps only small values and (key, first page, size) in memory; ``close`` sorts
    the keys and writes the leaves, the branch levels and the two meta pages.  A multiscale image set of ~100 GB therefore
    never sits in memory.  Fixture / export tool, not a transactional store: the file is complete only after ``close``."""

    def __init__(self, path, page_size=4096):
        os.makedirs(path, exist_ok=True)
        self.path = os.path.join(path, "data.mdb")
        self.page_size = page_size
        self.node_max = ((page_size - PAGE_HDR) // 2 - 2) & ~1        # mdb.c: me_nodemax
        self.entries = []                                                # (key, node payload, node flags, data size)
        self.overflow_pages = 0
        self.next_pg = 2
        self.f = open(self.path, "wb")
        self.f.write(bytes(2 * page_size))                               # the meta pages, written last

    def __enter__(self):
        return self

    def __exit__(self, exc_type, *_):
        if exc_type is None:
            self.close()
        else:
            self.f.close()

    def put(self, key, value):
        key = key if isinstance(key, bytes) else key.encode("utf-8")
        value = bytes(value)
        if len(key) > 511:
            raise ValueError("LMDB keys are at most 511 bytes")
        if NODE_HDR + len(key) + len(value) > self.node_max:
            n = (PAGE_HDR + len(value) + self.page_size - 1) // self.page_size
            pg = self.next_pg
            self.next_pg += n
            self.f.write(struct.pack("<QHHI", pg, 0, P_OVERFLOW, n) + value + bytes(n * self.page_size - PAGE_HDR - len(value)))
            self.overflow_pages += n
            self.entries.append((key, struct.pack("<Q", pg), F_BIGDATA, len(value)))
        else:
            self.entries.append((key, value, 0, len(value)))

    def _level(self, entries, leaf):
        """Write one tree level.  entries: leaf -> (key, node payload, node flags, data size); branch -> (key, child pgno).
        Returns [(first key, pgno)] of the pages written."""
        out, cur, used = [], [], 0
        page_size = self.page_size
        cap = page_size - PAGE_HDR

        def even(n):
            return (n + 1) & ~1

        def flush():
            nonlocal cur, used
            if not cur:
                return
            pgno = self.next_pg
            self.next_pg += 1
            page = bytearray(page_size)
            upper = page_size
            ptrs = []
            for idx, e in enumerate(cur):
                if leaf:
                    key, payload, nflags, dsize = e
                    lo, hi = dsize & 0xFFFF, dsize >> 16
                else:
                    key, child = e
                    if idx == 0:
                        key = b""                                  # a branch page's first separator is implicit
                    payload, lo, hi, nflags = b"", child & 0xFFFF, (child >> 16) & 0xFFFF, child >> 32
                node = struct.pack("<HHHH", lo, hi, nflags, len(key)) + key + payload
                upper -= even(len(node))
                page[upper:upper + len(node)] = node
                ptrs.append(upper)
            lower = PAGE_HDR + 2 * len(ptrs)
            assert lower <= upper
            struct.pack_into("<QHHHH", page, 0, pgno, 0, P_LEAF if leaf else P_BRANCH, lower, upper)
            struct.pack_into(f"<{len(ptrs)}H", page, PAGE_HDR, *ptrs)
            self.f.write(page)
            out.append((cur[0][0], pgno))
            cur, used = [], 0
        for e in entries:
            nsz = even(NODE_HDR + len(e[0]) + (len(e[1]) if leaf else 0)) + 2
            if used + nsz > cap:
                flush()
            cur.append(e)
            used += nsz
        flush()
        return out

    def close(self):
        """Sort the keys, write the tree and the meta pages; returns the path of data.mdb."""
        entries = sorted(self.entries, key=lambda e: e[0])
        for a, b in zip(entries, entries[1:]):
            if a[0] == b[0]:
                self.f.close()
                raise ValueError(f"duplicate key {a[0]!r}")
        level = self._level(entries, True)
        leaf_pages, branch_pages, depth = len(level), 0, 1 if level else 0
        while len(level) > 1:
            level = self._level(level, False)
            branch_pages += len(level)
            depth += 1
        root = level[0][1] if level else P_INVALID
        last_pg = self.next_pg - 1
        self.f.seek(0)
        for pg in (0, 1):
            page = bytearray(self.page_size)
            struct.pack_into("<QHHHH", page, 0, pg, 0, P_META, 0, 0)
            free_db = struct.pack("<IHHQQQQQ", self.page_size, 0, 0, 0, 0, 0, 0, P_INVALID)
            main_db = struct.pack("<IHHQQQQQ", 0, 0, depth, branch_pages, leaf_pages, self.overflow_pages, len(entries), root)
            meta = struct.pack("<IIQQ", MDB_MAGIC, MDB_VERSION, 0, max(1 << 20, (last_pg + 1) * self.page_size)) + free_db + \
                main_db + struct.pack("<QQ", last_pg, pg)              # txnid: page 1 is the newer one
            page[PAGE_HDR:PAGE_HDR + len(meta)] = meta
            self.f.write(page)
        self.f.close()
        return self.path


def write_lmdb(path, items, page_size=4096):
    """Bulk-write ``items`` (an iterable of (key bytes, value bytes)) as an LMDB environment directory ``path`` (data.mdb),
    through ``LmdbWriter`` in key order.  Returns the path of data.mdb."""
    items = sorted((k if isinstance(k, bytes) else k.encode("utf-8"), bytes(v)) for k, v in items)
    for (a, _), (b, _) in zip(items, items[1:]):
        if a == b:
            raise ValueError(f"duplicate key {a!r}")
    w = LmdbWriter(path, page_size)
    for k, v in items:
        w.put(k, v)
    return w.close()


# ---------------------------------------------------------------------------------------------- key schema / decode
def image_key(resolution, index):
    """prepare_ffhq_multiscale_dataset.py:58, dataset_loaders.py:252."""
    return f"{resolution}-{str(index).zfill(5)}".encode("utf-8")


def normal_map_key(resolution, index):
    """dataset_loaders.py:262."""
    return f"norm_map_{resolution}-{str(index).zfill(5)}".encode("utf-8")


def decode_image(data, resolution=None):
    """Encoded bytes -> float32 (3,H,W) in [-1,1]: PIL decode, optional resize (dataset_loaders.py:268-270,276-279),
    ``ToTensor`` + ``Normalize((0.5,)*3, (0.5,)*3)`` (dataset_loaders.py:128-137)."""
    from PIL import Image
    img = Image.open(io.BytesIO(data)).convert("RGB")
    if resolution is not None and img.size[0] != resolution:
        img = img.resize((resolution, resolution))
    a = np.asarray(img, dtype=np.float32)
    return torch.from_numpy(a).permute(2, 0, 1).div_(255.0).sub_(0.5).div_(0.5)


class GifLmdbDataset(torch.utils.data.Dataset):
    """The reference's FFHQ item for ``rendered_flame_as_condition=True, normal_maps_as_cond=True`` (dataset_loaders.py:236-330):
    ``(img (3,R,R), [cond (6,R,R)], [flame_label (P,)], index)``, all float32, images in [-1,1].

    ``rendered_flame_root=None``: there is no render LMDB; the conditions are rendered on the device from the raw parameter
    rows by ``DeviceBatchLoader(dataset, ..., conditions=DecaConditionRenderer(...))``, and indexing the dataset raises."""

    def __init__(self, real_img_root, rendered_flame_root, flame_params, resolution=256, rend_flm_res=256, valid_ids=None,
                 flame_mean=0.0, flame_std=1.0):
        self.real = LmdbReader(real_img_root)
        self.rend = None if rendered_flame_root is None else LmdbReader(rendered_flame_root)
        self.length = int(self.real.get(b"length").decode("utf-8"))           # dataset_loaders.py:168
        self.resolution, self.rend_flm_res = resolution, rend_flm_res
        self.flame_params = np.asarray(flame_params, dtype=np.float32)
        self.valid_ids = np.arange(self.length) if valid_ids is None else np.asarray(valid_ids)
        self.flame_mean, self.flame_std = flame_mean, flame_std

    def __len__(self):
        return len(self.valid_ids)

    def __getitem__(self, index):
        if self.rend is None:
            raise RuntimeError("this dataset has no render LMDB (rendered_flame_root=None): its conditions are rendered on the "
                               "device, so batches come from DeviceBatchLoader(dataset, ..., conditions=DecaConditionRenderer(...))")
        i = int(self.valid_ids[index])
        img = decode_image(self.real.get(image_key(self.resolution, i)))
        rnd = decode_image(self.rend.get(image_key(self.rend_flm_res, i)), self.resolution)
        nrm = decode_image(self.rend.get(normal_map_key(self.rend_flm_res, i)), self.resolution)
        lbl = (self.flame_params[i] - self.flame_mean) / self.flame_std
        return img, [torch.cat((rnd, nrm), 0)], [torch.from_numpy(np.asarray(lbl, dtype=np.float32))], i


class PinnedBatchLoader:
    """Batches of a GifLmdbDataset assembled in PINNED host memory by a background thread (decode is host work; the copy to the
    device is one non-blocking transfer per tensor, issued by the trainer).  Yields (real (B,3,R,R), cond (B,6,R,R),
    labels (B,P), indices (B,) int64) -- the arguments of ``GifTrainer.train_iteration``; ``depth`` batches are in flight."""

    def __init__(self, dataset, batch_size, shuffle=True, seed=0, depth=3, pin=None):
        self.ds, self.bs, self.shuffle, self.seed, self.depth = dataset, batch_size, shuffle, seed, depth
        self.pin = torch.cuda.is_available() if pin is None else pin
        img, cond, lbl, _ = dataset[0]
        self._shapes = (tuple(img.shape), tuple(cond[0].shape), tuple(lbl[0].shape))

    def _alloc(self):
        mk = (lambda *s, dtype=torch.float32: torch.empty(*s, dtype=dtype).pin_memory()) if self.pin else \
            (lambda *s, dtype=torch.float32: torch.empty(*s, dtype=dtype))
        return (mk(self.bs, *self._shapes[0]), mk(self.bs, *self._shapes[1]), mk(self.bs, *self._shapes[2]),
                mk(self.bs, dtype=torch.int64))

    def __iter__(self):
        order = np.arange(len(self.ds))
        if self.shuffle:
            np.random.default_rng(self.seed).shuffle(order)
            self.seed += 1
        nb = len(order) // self.bs                                              # drop_last=True, dataset_loaders.py:395
        free, ready = queue.Queue(), queue.Queue(maxsize=self.depth)
        for _ in range(self.depth + 1):
            free.put(self._alloc())

        def work():
            for b in range(nb):
                buf = free.get()
                for j, idx in enumerate(order[b * self.bs:(b + 1) * self.bs]):
                    img, cond, lbl, i = self.ds[int(idx)]
                    buf[0][j].copy_(img); buf[1][j].copy_(cond[0]); buf[2][j].copy_(lbl[0]); buf[3][j] = i
                ready.put(buf)
            ready.put(None)
        threading.Thread(target=work, daemon=True).start()
        while True:
            buf = ready.get()
            if buf is None:
                return
            yield buf
            free.put(buf)       # the consumer is done with the previous batch once it asks for the next one


class DeviceBatchLoader:
    """Batches of a GifLmdbDataset decoded on the device (gif_b200.image_decode), bitwise equal to ``PinnedBatchLoader``'s
    with the same order, seed handling and drop_last.  Real images must be baseline JPEG and renders 8-bit PNG, as the
    reference's LMDB writers store them; anything else raises ``UnsupportedImage`` naming the key.

    A background thread reads the raw LMDB values, parses them, inflates the PNGs on a small thread pool and packs them as
    one ``image_decode.DecodeBatch`` (a pinned byte arena).  The consuming thread enqueues its decode on a side stream,
    one batch ahead, so batch k+1 decodes while the caller trains on batch k.  It yields device tensors (real (B,3,R,R),
    cond (B,6,R,R), labels (B,P), indices (B,) int64) -- the arguments of ``GifTrainer.train_iteration`` -- after making the
    current stream wait for their decode.  Each batch stays valid until the next one is requested.  Before yielding a batch
    it waits for that batch's decode (queued a step earlier on the side stream, never behind training work) and reads its
    per-image status words, so a corrupt image raises before its batch is used.

    ``conditions``: a ``gif_b200.conditions.DecaConditionRenderer`` at the dataset's ``rend_flm_res``.  The conditions are
    then rendered on the side stream from the raw parameter rows (``dataset.flame_params``), which travel with the labels;
    no render key is read and nothing is inflated.  The rendered bytes are what the reference's render LMDB holds, so the
    batches equal those of the LMDB path wherever the rasteriser agrees with the one that wrote it."""

    def __init__(self, dataset, batch_size, shuffle=True, seed=0, depth=3, device=None, threads=4, conditions=None):
        self.ds, self.bs, self.shuffle, self.seed, self.depth = dataset, batch_size, shuffle, seed, depth
        self.device = torch.device(device or "cuda")
        self.threads = threads
        if conditions is not None and conditions.image_size != dataset.rend_flm_res:
            raise ValueError(f"the condition renderer draws {conditions.image_size}^2, the dataset's rend_flm_res is "
                             f"{dataset.rend_flm_res}")
        if conditions is not None and dataset.flame_params.shape[-1] < 236:
            raise ValueError(f"rendering conditions needs DECA rows of at least 236 columns, the dataset's parameter table "
                             f"has {dataset.flame_params.shape[-1]}")
        if conditions is None and dataset.rend is None:
            raise ValueError("the dataset has no render LMDB (rendered_flame_root=None): pass conditions=DecaConditionRenderer(...)")
        self.conditions = conditions
        self.pin = torch.cuda.is_available()
        self._stream = None

    def host_batch(self, ids, pool):
        """The host side of one batch, run on the loader's thread: the LMDB reads, the JPEG parsing and, on ``pool``, the PNG
        inflate, packed as one ``image_decode.DecodeBatch`` (real images, then renders, then normal maps); the labels,
        indices and, when rendering, the raw parameter rows.  Real images must be JPEG at the dataset's resolution and
        renders PNG at its rend_flm_res."""
        from . import image_decode as I
        ds, R, rr = self.ds, self.ds.resolution, self.ds.rend_flm_res
        render = self.conditions is not None

        def load(db, key, kind, size):
            im = I.host_decode(db.get(key), key.decode())
            if im.kind != kind or (im.w, im.h) != (size, size):
                raise I.UnsupportedImage(f"{im.name}: a {im.w}x{im.h} {im.kind.upper()}; the dataset's "
                                         f"{'renders' if kind == 'png' else 'real images'} are {size}x{size} {kind.upper()}s")
            return im
        rkeys = [] if render else [image_key(rr, i) for i in ids] + [normal_map_key(rr, i) for i in ids]
        pngs = pool.map(lambda k: load(ds.rend, k, "png", rr), rkeys)   # inflates while this thread parses the JPEGs
        jpegs = [load(ds.real, image_key(R, i), "jpeg", R) for i in ids]
        batch = I.DecodeBatch(jpegs + list(pngs))
        lbl = np.stack([(ds.flame_params[i] - ds.flame_mean) / ds.flame_std for i in ids]).astype(np.float32)
        pin = (lambda t: t.pin_memory()) if self.pin else (lambda t: t)
        # the renderer takes the raw rows: (p - m) / s * s + m is not p in float32
        raw = pin(torch.from_numpy(np.ascontiguousarray(ds.flame_params[ids], dtype=np.float32))) if render else None
        return batch, pin(torch.from_numpy(lbl)), pin(torch.tensor(ids, dtype=torch.int64)), raw

    def _launch(self, hb):
        """Enqueue the copy and the decode of one host batch on the side stream."""
        from . import image_decode as I
        batch, lbl, idx, raw = hb
        dev, B, R, rr = self.device, self.bs, self.ds.resolution, self.ds.rend_flm_res
        with torch.cuda.stream(self._stream):
            images, status = batch.decode(dev)
            real_u8 = I.as_batch(images[:B])
            if raw is None:
                rend_u8 = I.as_batch(images[B:])
            else:
                rend_u8 = torch.empty(2 * B, rr, rr, 3, dtype=torch.uint8, device=dev)
                self.conditions.render_u8(raw.to(dev, non_blocking=True), out=rend_u8)
            if rr != R:
                rend_u8 = I.resize_bicubic_u8(rend_u8, R)
            real = torch.empty(B, 3, R, R, device=dev)
            cond = torch.empty(B, 6, R, R, device=dev)
            I.u8_to_unit(real_u8, real)
            I.u8_to_unit(rend_u8[:B], cond[:, 0:3])
            I.u8_to_unit(rend_u8[B:], cond[:, 3:6])
            labels, indices = lbl.to(dev, non_blocking=True), idx.to(dev, non_blocking=True)
            st = status.to("cpu", non_blocking=True) if self.pin else status.cpu()
            done = torch.cuda.Event()
            done.record()
        return (real, cond, labels, indices), st, done, batch.names

    def _finish(self, launched):
        from . import image_decode as I
        out, st, done, names = launched
        done.synchronize()                          # the side stream only: this batch's copy and decode
        I.check_status(st, names)
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(done)
        for t in out:                               # allocated on the side stream, used on this one
            t.record_stream(cur)
        return out

    def __iter__(self):
        order = np.arange(len(self.ds))
        if self.shuffle:
            np.random.default_rng(self.seed).shuffle(order)
            self.seed += 1
        nb = len(order) // self.bs                                              # drop_last=True, dataset_loaders.py:395
        if self._stream is None:
            self._stream = torch.cuda.Stream(self.device)
        ready = queue.Queue(maxsize=self.depth)
        stop = threading.Event()

        def work():
            from concurrent.futures import ThreadPoolExecutor
            with ThreadPoolExecutor(self.threads) as pool:
                for b in range(nb):
                    if stop.is_set():
                        return
                    ids = [int(self.ds.valid_ids[int(j)]) for j in order[b * self.bs:(b + 1) * self.bs]]
                    try:
                        item = self.host_batch(ids, pool)
                    except Exception as e:          # handed to the consumer, which raises it
                        item = e
                    ready.put(item)
                    if isinstance(item, Exception):
                        return
            ready.put(None)

        def next_launched():
            hb = ready.get()
            if isinstance(hb, Exception):
                raise hb
            return None if hb is None else self._launch(hb)
        threading.Thread(target=work, daemon=True).start()
        try:
            pending = next_launched()
            while pending is not None:
                ahead = next_launched()             # batch k+1 decodes on the side stream while batch k trains
                yield self._finish(pending)
                pending = ahead
        finally:
            stop.set()
            while not ready.empty():
                ready.get_nowait()
