"""CPU: the host side of the real images' FID statistics (gif_b200/fid_real.py): which files are used (the reference's
rules with sorted names), which PNGs are rejected, the atomic cache write, and ``FidComputer.compute_true_img_response``
choosing between the cache, the image folder and an error."""
import os

import numpy as np
import pytest
import torch

from gif_b200 import fid, fid_real
from gif_b200.image_decode import UnsupportedImage
from gif_b200.synth_images import noise, png, png_chunks


def touch(d, names):
    for n in names:
        (d / n).write_bytes(b"")


def test_files_sorted_png_only(tmp_path):
    touch(tmp_path, ["b.png", "a.png", "c.PNG", "d.jpg", ".hidden.png", "e.png.bak", "f.png"])
    (tmp_path / "sub").mkdir()
    touch(tmp_path / "sub", ["g.png"])
    got = fid_real.real_image_files(tmp_path, batch_size=32)
    assert got == [str(tmp_path / n) for n in ("a.png", "b.png", "f.png")]


def test_files_whole_batches_and_small_folders(tmp_path):
    names = [f"{i:05d}.png" for i in range(70)]
    touch(tmp_path, names[::-1])
    got = fid_real.real_image_files(tmp_path)
    assert got == [str(tmp_path / n) for n in names[:64]]                # 70 // 32 batches: the remainder of 6 dropped
    assert len(fid_real.real_image_files(tmp_path, batch_size=10)) == 70
    assert len(fid_real.real_image_files(tmp_path, limit=32)) == 32
    assert fid_real.real_image_files(tmp_path, limit=20) == [str(tmp_path / n) for n in names[:20]]   # < 32: one batch
    assert len(fid_real.real_image_files(tmp_path, batch_size=100)) == 70


def test_files_capped_at_50000(tmp_path):
    names = [f"{i:05d}.png" for i in range(50_040)]
    touch(tmp_path, names)
    got = fid_real.real_image_files(tmp_path)
    assert len(got) == 50_000 - 50_000 % 32 and got[-1] == str(tmp_path / names[len(got) - 1])


def test_no_files(tmp_path):
    touch(tmp_path, ["a.jpg"])
    with pytest.raises(FileNotFoundError, match="no \\*.png"):
        fid_real.real_image_files(tmp_path)


def test_rgb_png_loads(tmp_path):
    p = tmp_path / "ok.png"
    a = np.asarray(noise(5, 7, 1))
    p.write_bytes(png(noise(5, 7, 1)))
    (w, h, bpp, _), raw = fid_real.load_png(str(p))
    assert (w, h, bpp) == (7, 5, 3) and len(raw) == 5 * (1 + 7 * 3) and a.shape == (5, 7, 3)


@pytest.mark.parametrize("kind", ["grey", "grey_alpha", "rgba", "palette", "16bit", "interlaced"])
def test_non_rgb8_rejected_with_the_file_named(tmp_path, kind):
    from PIL import Image
    rgb = np.asarray(noise(4, 6, 2))
    if kind == "grey":
        blob = png(noise(4, 6, 2, "L"))
    elif kind == "grey_alpha":
        blob = png(Image.fromarray(rgb[..., :2].copy(), "LA"))
    elif kind == "rgba":
        blob = png(noise(4, 6, 2, "RGBA"))
    elif kind == "palette":
        blob = png(noise(4, 6, 2).convert("P"))
    elif kind == "16bit":
        blob = png_chunks(6, 4, 2, b"".join(b"\0" + bytes(6 * 6) for _ in range(4)), depth=16)
    else:
        blob = png_chunks(6, 4, 2, b"".join(b"\0" + bytes(6 * 3) for _ in range(4)), interlace=1)
    p = tmp_path / f"img_{kind}.png"
    p.write_bytes(blob)
    with pytest.raises(UnsupportedImage, match=f"img_{kind}.png"):
        fid_real.load_png(str(p))


def test_statistics_need_a_cuda_device(tmp_path):
    touch(tmp_path, ["a.png"])
    with pytest.raises(RuntimeError, match="CUDA"):
        fid_real.real_image_statistics(tmp_path, 256, torch.nn.Identity(), 8, device="cpu")


def test_cache_written_atomically(tmp_path, monkeypatch):
    p = str(tmp_path / "stats" / "ffhq_256X256_fid_stats.npz")
    mu, sigma = np.arange(4.0), np.eye(4) * 0.5
    fid_real.save_statistics(p, mu, sigma)
    f = np.load(p)
    assert f["mu"].dtype == np.float64 and np.array_equal(f["mu"][:], mu) and np.array_equal(f["sigma"][:], sigma)
    f.close()
    assert os.listdir(os.path.dirname(p)) == [os.path.basename(p)]

    def broken(fh, **kw):                                     # a write that dies half way: the old cache stays
        fh.write(b"PK partial")
        raise OSError("disk full")
    monkeypatch.setattr(np, "savez", broken)
    with pytest.raises(OSError, match="disk full"):
        fid_real.save_statistics(p, mu + 1, sigma)
    monkeypatch.undo()
    with np.load(p) as f:
        assert np.array_equal(f["mu"][:], mu)
    assert os.listdir(os.path.dirname(p)) == [os.path.basename(p)]


class _Feat(torch.nn.Module):
    def forward(self, x):
        return [x]


def test_true_img_response_cache_folder_or_error(tmp_path, monkeypatch):
    calls = []

    def fake_stats(root, resolution, model, dims, device=None, **kw):
        calls.append((root, resolution, dims))
        return torch.arange(3, dtype=torch.float64), torch.eye(3, dtype=torch.float64) * 2

    monkeypatch.setattr(fid_real, "real_image_statistics", fake_stats)
    stats_dir = tmp_path / "stats"
    fc = fid.FidComputer(database_root_dir=str(tmp_path / "imgs"), true_img_stats_dir=str(stats_dir), model=_Feat(), dims=3,
                         device=torch.device("cpu"))
    fc.compute_true_img_response(64)
    assert calls == [(str(tmp_path / "imgs"), 64, 3)]
    with np.load(stats_dir / "ffhq_64X64_fid_stats.npz") as f:
        assert np.array_equal(f["mu"][:], [0.0, 1.0, 2.0]) and np.array_equal(f["sigma"][:], np.eye(3) * 2)
    fc2 = fid.FidComputer(database_root_dir=None, true_img_stats_dir=str(stats_dir), model=_Feat(), dims=3,
                          device=torch.device("cpu"))
    fc2.compute_true_img_response(64)                         # the cache: no computation
    assert len(calls) == 1 and np.array_equal(fc2.s_t, np.eye(3) * 2)

    monkeypatch.chdir(tmp_path)
    fc3 = fid.FidComputer(database_root_dir=str(tmp_path / "imgs"), true_img_stats_dir=None, model=_Feat(), dims=3,
                          device=torch.device("cpu"))
    fc3.compute_true_img_response(32)                         # computed, not written
    assert len(calls) == 2 and np.array_equal(fc3.m_t, [0.0, 1.0, 2.0])
    assert sorted(os.listdir(tmp_path)) == ["stats"]

    fc4 = fid.FidComputer(true_img_stats_dir=str(stats_dir), model=_Feat(), dims=3, device=torch.device("cpu"))
    with pytest.raises(FileNotFoundError, match="ffhq_32X32_fid_stats.npz"):
        fc4.compute_true_img_response(32)
