"""CPU: the facts the device-rendered conditions rest on -- the reference's render quantisation survives its uint8 / PNG round
trip exactly, and the loader's [-1,1] mapping of those bytes is bitwise the render's own quantised condition -- plus the
DECA column layout and the errors of the render-fed data path."""
import io

import numpy as np
import pytest
import torch
from PIL import Image


def _levels():
    """float32 inputs hitting every quantisation level from below, on and just above it, and out of range."""
    base = np.arange(256, dtype=np.float32)
    frac = np.array([0.0, 1e-4, 0.25, 0.5, 0.999], np.float32)
    t = (base[:, None] + frac[None]).ravel()
    return np.concatenate([t, np.float32([-3.0, -1e-6, 255.5, 300.0])]).astype(np.float32)


def test_quantisation_survives_the_lmdb_round_trip():
    """visualize_flame_overlay.py:29-31 then create_deca_rendered_lmdb.py:67-70 (x*255).astype('uint8') and a PNG, then
    ToTensor + Normalize, against floor(clamp) and the render's q*2-1 epilogue -- for all 256 levels."""
    t = torch.from_numpy(_levels())
    n = t / 255.0 * 1.05 - 0.02                                               # normal components, also outside [0,1]
    q_t = torch.floor(t.clamp(0, 255)) / 255.0
    q_n = torch.floor(n.clamp(0, 1) * 255) / 255.0
    for q, direct in ((q_t, torch.floor(t.clamp(0, 255))), (q_n, torch.floor(n.clamp(0, 1) * 255))):
        u8 = (q.numpy() * 255).astype("uint8")
        assert np.array_equal(u8, direct.numpy().astype(np.uint8))           # what cond_u8 writes
        side = int(np.ceil(np.sqrt(u8.size / 3)))
        ramp = np.zeros(side * side * 3, np.uint8)
        ramp[:u8.size] = u8
        buf = io.BytesIO()
        Image.fromarray(ramp.reshape(side, side, 3)).save(buf, format="png", quality=100)
        back = np.asarray(Image.open(io.BytesIO(buf.getvalue())).convert("RGB")).ravel()[:u8.size]
        assert np.array_equal(back, u8)
        unit = (torch.from_numpy(back.astype(np.float32)) / 255.0 - 0.5) / 0.5  # u8_to_unit
        assert torch.equal(unit, q.clamp(0, 1) * 2 - 1)                       # the render_shade cond epilogue
    assert sorted(set(np.floor(_levels().clip(0, 255)).astype(int))) == list(range(256))


def test_deca_slicing_follows_the_reference_layout():
    from gif_b200.conditions import DECA_COLUMNS, DECA_SLICES, split_deca
    # constants.INDICES (SHAPE, EXP, POSE, TRANS) and constants.DECA_IDX (cam, tex, lit) of the reference
    indices = {"SHAPE": (0, 100), "EXP": (100, 150), "POSE": (150, 156), "TRANS": (156, 159)}
    deca_idx = {"cam": (156, 159), "tex": (159, 209), "lit": (209, 236)}
    assert (DECA_SLICES["shape"], DECA_SLICES["exp"], DECA_SLICES["pose"]) == \
        (indices["SHAPE"], indices["EXP"], indices["POSE"])
    assert DECA_SLICES["cam"] == indices["TRANS"] == deca_idx["cam"]
    assert DECA_SLICES["tex"] == deca_idx["tex"] and DECA_SLICES["lit"] == deca_idx["lit"]
    assert DECA_COLUMNS == deca_idx["lit"][1]
    rows = torch.arange(3 * 240, dtype=torch.float32).reshape(3, 240)
    p = split_deca(rows)
    for k, (a, b) in DECA_SLICES.items():
        assert torch.equal(p[k].reshape(3, -1), rows[:, a:b]), k
    assert p["lit"].shape == (3, 9, 3) and torch.equal(p["lit"][:, 1, 0], rows[:, 212])       # (9,3) row-major


def test_short_parameter_table_raises():
    from gif_b200.conditions import split_deca
    with pytest.raises(ValueError, match="159"):
        split_deca(torch.zeros(4, 159))


def _dataset(tmp_path, params, rend=False):
    from gif_b200.data import GifLmdbDataset
    from gif_b200.synth_images import build_lmdbs
    real, rend_root = build_lmdbs(tmp_path, len(params), 32, 32)
    return GifLmdbDataset(real, rend_root if rend else None, params, resolution=32, rend_flm_res=32)


def test_dataset_without_render_lmdb_points_at_the_device_loader(tmp_path):
    from gif_b200.data import DeviceBatchLoader, PinnedBatchLoader
    ds = _dataset(tmp_path, np.zeros((4, 236), np.float32))
    assert len(ds) == 4
    with pytest.raises(RuntimeError, match=r"DeviceBatchLoader\(.*conditions="):
        ds[0]
    with pytest.raises(RuntimeError, match="conditions="):
        PinnedBatchLoader(ds, 2)
    with pytest.raises(ValueError, match="conditions="):
        DeviceBatchLoader(ds, 2)


def test_device_loader_checks_the_renderer_against_the_dataset(tmp_path):
    from gif_b200.data import DeviceBatchLoader

    class Renderer:                                  # the loader only needs image_size before the first batch
        image_size = 32
    with pytest.raises(ValueError, match="159"):
        DeviceBatchLoader(_dataset(tmp_path / "a", np.zeros((4, 159), np.float32)), 2, conditions=Renderer())
    Renderer.image_size = 64
    with pytest.raises(ValueError, match="rend_flm_res"):
        DeviceBatchLoader(_dataset(tmp_path / "b", np.zeros((4, 236), np.float32)), 2, conditions=Renderer())
