"""GPU: conditions rendered on the device from DECA rows (gif_b200.conditions) -- FLAMETex against the reference's own
module, deterministic vertex normals, the uint8 render output against the float condition, and DeviceBatchLoader fed by
the renderer yielding bitwise the batches it yields from an LMDB written the way prepare_lmdb/create_deca_rendered_lmdb.py
writes one."""
import io
import math

import numpy as np
import pytest
import torch
from PIL import Image

import golden_util as gu
from gif_b200.flame_synth import synthetic_deca_params

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def space():
    from gif_b200.flame_synth import synthetic_texture_space
    return synthetic_texture_space(512, 50)


@pytest.fixture(scope="module")
def parts(cuda, space):
    from gif_b200.flame import FLAME, FLAMETex
    from gif_b200.flame_synth import flame_uv, synthetic_flame_model
    flame = FLAME.from_arrays(synthetic_flame_model()).to(cuda)
    tex = FLAMETex(mean=space[0], basis=space[1]).to(cuda)
    uv, uvf = flame_uv()
    return flame, tex, uv, uvf


def renderer(parts, size):
    from gif_b200.conditions import DecaConditionRenderer
    return DecaConditionRenderer(*parts, image_size=size)


def test_flametex_matches_reference_golden(cuda, space):
    """oracle/make_flametex_golden.py: the reference's FLAMETex on the same analytic texture space (side 512, n 50)."""
    from gif_b200.flame import FLAMETex
    g = gu.load_golden("flametex.npz")
    tex = FLAMETex(mean=space[0], basis=space[1]).to(cuda)
    code = torch.from_numpy(g["texcode"]).to(cuda)
    out = tex(code)
    assert tuple(out.shape) == (code.shape[0], 3, 256, 256)
    got = out.cpu().numpy()[tuple(g["index"].astype(np.int64).T)]
    assert np.abs(got - g["albedo"]).max() <= 1e-5 * float(g["albedo_abs_max"])
    # more texcodes than one staging pass (32) and a ragged tail: every image is computed the same way
    big = tex(code.repeat(10, 1)[:37])
    for i in range(37):
        assert torch.equal(big[i], out[i % 4]), i


def test_vertex_normals_deterministic(cuda):
    from gif_b200.flame_synth import flame_topology, synthetic_flame_params
    from gif_b200.render import vertex_normals
    verts = synthetic_flame_params(3, seed=4)[0]
    _, faces = flame_topology()
    v = torch.cat([verts, verts[1:2], verts[0:1]]).to(cuda)                    # images 3, 4 repeat images 1, 0
    a, fa = vertex_normals(v, faces.to(cuda), face_normals=True)
    b = vertex_normals(v, faces.to(cuda))
    assert torch.equal(a, b)
    assert torch.equal(a[3], a[1]) and torch.equal(a[4], a[0])
    assert torch.equal(fa, a[:, faces.to(cuda)])


@pytest.mark.parametrize("size", [64, 256])
def test_u8_render_maps_to_the_float_condition(cuda, parts, size):
    cr = renderer(parts, size)
    deca = synthetic_deca_params(5, 1, cols=240).to(cuda)
    cond = cr(deca)
    u8 = cr.render_u8(deca)
    flame, tex = parts[:2]
    verts, _ = flame.decode_vertices(deca[:, 0:100].contiguous(), deca[:, 100:150].contiguous(), deca[:, 150:156].contiguous())
    want = cr.renderer.render_tex_and_normal(verts, deca[:, 156:159].contiguous(), tex(deca[:, 159:209]),
                                             deca[:, 209:236].reshape(-1, 9, 3))[2]
    assert torch.equal(cond, want)
    assert tuple(u8.shape) == (10, size, size, 3) and torch.equal(cr.render_u8(deca), u8)
    assert 0.2 < float((u8[5:] > 0).any(-1).float().mean()) < 0.95                 # a head, not an empty frame
    with pytest.raises(ValueError, match="159"):
        cr.render_u8(deca[:, :159])


def write_render_lmdb(path, cr, deca, ids):
    """create_deca_rendered_lmdb.py:53-89 on our renderer: get_rendered_mesh's quantisation, (x*255).astype('uint8'),
    Pillow PNG, one key per image and normal map."""
    from gif_b200.data import image_key, normal_map_key, write_lmdb
    from gif_b200.render import batch_orth_proj
    flame, tex = cr.flame, cr.flametex
    verts, _ = flame.decode_vertices(deca[:, 0:100].contiguous(), deca[:, 100:150].contiguous(), deca[:, 150:156].contiguous())
    trans = batch_orth_proj(verts, deca[:, 156:159].contiguous())
    trans[:, :, 1:] = -trans[:, :, 1:]
    out = cr.renderer(verts, trans, tex(deca[:, 159:209]), deca[:, 209:236].reshape(-1, 9, 3), want_cond=False)
    textured = torch.floor(out["images"].clamp(0, 255)) / 255.0                # visualize_flame_overlay.py:29-31
    normal = torch.floor(out["normal_images"].clamp(0, 1) * 255) / 255.0
    items = []
    for j, i in enumerate(ids):
        for key, img in ((image_key(cr.image_size, i), textured[j]), (normal_map_key(cr.image_size, i), normal[j])):
            buf = io.BytesIO()
            Image.fromarray((img.cpu().numpy() * 255).astype("uint8").transpose((1, 2, 0))).save(buf, format="png", quality=100)
            items.append((key, buf.getvalue()))
    write_lmdb(path, items)
    return path


@pytest.mark.parametrize("R,rr", [(64, 64), (128, 64)])
def test_render_fed_loader_equals_lmdb_fed_loader(cuda, parts, tmp_path, R, rr):
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset
    from gif_b200.synth_images import build_lmdbs
    n, bs = 12, 4
    cr = renderer(parts, rr)
    params = synthetic_deca_params(n, 7).numpy()
    real, _ = build_lmdbs(tmp_path, n, R, rr)
    rend = write_render_lmdb(str(tmp_path / "deca_rend"), cr, torch.from_numpy(params).to(cuda), list(range(n)))
    kw = dict(resolution=R, rend_flm_res=rr, flame_mean=0.25, flame_std=1.5)
    from_lmdb = DeviceBatchLoader(GifLmdbDataset(real, rend, params, **kw), bs, seed=3)
    rendered = DeviceBatchLoader(GifLmdbDataset(real, None, params, **kw), bs, seed=3, conditions=cr)
    for _epoch in range(2):
        count = 0
        for a, b in zip(from_lmdb, rendered):
            for x, y in zip(a, b):
                assert y.is_cuda and torch.equal(x, y)
            count += 1
        assert count == n // bs


def test_trainer_fed_by_render_loader(cuda, parts, tmp_path):
    from gif_b200 import ops
    from gif_b200.data import DeviceBatchLoader, GifLmdbDataset
    from gif_b200.synth_images import build_lmdbs
    from gif_b200.train_step import GifTrainer
    ops.set_precision("tf32")
    res, b, n = 32, 4, 8
    real, _ = build_lmdbs(tmp_path, n, res, res)
    ds = GifLmdbDataset(real, None, synthetic_deca_params(n, 9).numpy(), resolution=res, rend_flm_res=res)
    loader = DeviceBatchLoader(ds, b, seed=1, conditions=renderer(parts, res))
    tr = GifTrainer(cuda, res, vocab=16, r1_every=2, ppl=False, seed=3)
    losses = []
    for epoch in range(2):
        for real_b, cond_b, _, idx_b in loader:
            losses.append([float(v) for v in tr.train_iteration(real_b, cond_b, idx_b % 16)])
        if epoch == 0:
            tr.capture(b, res)
    assert len(losses) == 4 and all(math.isfinite(v) for row in losses for v in row), losses
