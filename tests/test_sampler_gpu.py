"""GPU: generating faces from FLAME parameters (gif_b200.eye_centering, gif_b200.sampler) -- the eye-camera kernel against
the float64 restatement and the unmodified reference's golden, the image-bytes kernel against numpy's float32 formula,
and FlameSampler against the composition of the existing public pieces, graph replay against eager, and batch
independence (the premise of padding a short last batch)."""
import numpy as np
import pytest
import torch

import golden_util as gu
from gif_b200.flame_synth import synthetic_deca_params
from oracle import eye_centering_oracle as EO

pytestmark = pytest.mark.gpu
VOCAB = 16


@pytest.fixture(scope="module")
def parts(cuda):
    from gif_b200.flame import FLAME, FLAMETex
    from gif_b200.flame_synth import flame_uv, synthetic_flame_model, synthetic_texture_space
    mean, basis = synthetic_texture_space(512, 50)
    flame = FLAME.from_arrays(synthetic_flame_model()).to(cuda)
    return flame, FLAMETex(mean=mean, basis=basis).to(cuda), *flame_uv()


@pytest.fixture(scope="module")
def cr(parts):
    from gif_b200.conditions import DecaConditionRenderer
    return DecaConditionRenderer(*parts, image_size=256)


@pytest.fixture()
def precision():
    from gif_b200 import ops
    old = ops.get_precision()
    yield ops.set_precision
    ops.set_precision(old)


def generator(cuda, seed=1):
    from gif_b200.model.stg2_generator import StyledGenerator
    G = StyledGenerator(embedding_vocab_size=VOCAB, rendered_flame_ascondition=True, normal_maps_as_cond=True)
    G.load_state_dict(gu.seeded_state_dict(gu.g_shapes(VOCAB), seed))
    return G.to(cuda).eval()


def np_bytes(x):
    """save_set_of_images' bytes of a clamped float32 NCHW batch, as the sampling scripts make them (numpy float32)."""
    x = np.clip(np.asarray(x, np.float32), -1, 1)
    return (np.clip((x + 1) / 2, 0, 1) * 255).astype(np.uint8).transpose(0, 2, 3, 1)


def rows_and_ids(n, seed, cuda):
    g = torch.Generator().manual_seed(seed)
    return synthetic_deca_params(n, seed).to(cuda), torch.randint(0, VOCAB, (n,), generator=g).to(cuda)


# ------------------------------------------------------------------------------------------------------- eye camera
def test_eye_camera_kernel_vs_float64_restatement(cuda):
    from gif_b200.eye_centering import EYE_TARGETS, eye_camera
    g = gu.load_golden("eye_centering.npz")
    assert np.array_equal(np.float32(EYE_TARGETS), g["targets"])
    cam = eye_camera(torch.from_numpy(g["eyes"]).to(cuda), eye_vertices=(0, 1)).cpu().numpy()
    want = EO.eye_camera(g["eyes"][:, 0], g["eyes"][:, 1])
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    assert (np.abs(cam - want) <= ulp).all(), np.abs(cam - want).max(0)
    d_ref = np.abs(cam - g["cam_ref"]).max(0)
    print(f"eye camera kernel vs the reference's float32 pinverse: max abs (scale, tx, ty) = {d_ref}")
    assert (d_ref <= g["pinv_err"] + np.spacing(np.abs(g["cam_ref"]).max(0))).all()


def test_eye_placement(cuda):
    """The fitted camera puts the midpoint of the two projected eyes (tests/test_eye_positioning.py:63-72 of the
    reference: (e + cam[1:]) * cam[0], y negated) on the target midpoint; x comes out mirrored by the scale's sign."""
    from gif_b200.eye_centering import EYE_TARGETS, eye_camera
    g = gu.load_golden("eye_centering.npz")
    eyes = g["eyes"]
    cam = eye_camera(torch.from_numpy(eyes).to(cuda), eye_vertices=(0, 1)).cpu().numpy()
    mid = EO.projected_eyes(eyes[:, 0], eyes[:, 1], cam).mean(1)
    x1, x2, y1, y2 = EYE_TARGETS
    scale = np.abs(cam[:, :1]) * (np.abs(eyes[:, :, :2]).max(1) + np.abs(cam[:, 1:]))
    tol = 8 * np.finfo(np.float32).eps * scale
    assert (np.abs(mid - np.array([-(x1 + x2) / 2, (y1 + y2) / 2])) <= tol).all()


def test_position_to_given_location_in_place(cuda, parts):
    from gif_b200.eye_centering import eye_camera, position_to_given_location
    flame = parts[0]
    g = gu.load_golden("eye_centering.npz")
    rows = torch.from_numpy(g["rows"]).to(cuda)
    before = rows.clone()
    out = position_to_given_location(flame, rows)
    assert out is rows
    assert torch.equal(rows[:, :156], before[:, :156]) and torch.equal(rows[:, 159:], before[:, 159:])
    verts, _ = flame.decode_vertices(before[:, :100].contiguous(), before[:, 100:150].contiguous(), before[:, 150:156].contiguous())
    assert torch.equal(rows[:, 156:159], eye_camera(verts))
    # the golden was decoded by the float32 CPU oracle; this decoder rounds differently (a few float32 ulps of the vertices),
    # and the camera moves by what that difference moves the float64 solution -- on top of the reference's pinverse error
    i1, i2 = EO.EYE_VERTICES
    eyes = verts[:, [i1, i2]].cpu().numpy()
    assert np.abs(eyes - g["eyes"]).max() < 2e-6
    decoder = np.abs(EO.eye_camera(eyes[:, 0], eyes[:, 1]) - EO.eye_camera(g["eyes"][:, 0], g["eyes"][:, 1])).max(0)
    err = np.abs(rows[:, 156:159].cpu().numpy() - g["cam_ref"]).max(0)
    print(f"position_to_given_location vs the reference golden: max abs (scale, tx, ty) = {err}; decoder term {decoder}")
    assert (err <= g["pinv_err"] + decoder + np.spacing(np.abs(g["cam_ref"]).max(0))).all(), (err, g["pinv_err"], decoder)


# ------------------------------------------------------------------------------------------------------ image bytes
def test_image_to_u8_bitwise(cuda):
    from gif_b200.image_decode import image_to_u8
    g = torch.Generator().manual_seed(3)
    rand = (torch.rand(4, 3, 32, 48, generator=g) * 3 - 1.5).numpy()
    levels = (2 * np.arange(256, dtype=np.float32) / np.float32(255) - 1).astype(np.float32)
    near = [levels]
    for k in (1, 2, 3):
        up, down = levels.copy(), levels.copy()
        for _ in range(k):
            up, down = np.nextafter(up, np.float32(2)), np.nextafter(down, np.float32(-2))
        near += [up, down]
    edge = np.concatenate(near + [np.float32([-1, 1, -1.0000001, 1.0000001, 0, -0.0, 5, -5])])
    edge = np.resize(edge, 3 * 8 * 64).reshape(1, 3, 8, 64).astype(np.float32)
    for x in (rand, edge):
        got = image_to_u8(torch.from_numpy(x).to(cuda)).cpu().numpy()
        assert np.array_equal(got, np_bytes(x))
    # the generator's output layout: an NCHW view of channels-last storage, and a strided crop of it
    nhwc = torch.from_numpy(rand).permute(0, 2, 3, 1).contiguous().to(cuda)
    view = nhwc.permute(0, 3, 1, 2)
    assert not view.is_contiguous()
    assert np.array_equal(image_to_u8(view).cpu().numpy(), np_bytes(rand))
    crop = view[1:, :, ::2, 3::3]
    assert np.array_equal(image_to_u8(crop).cpu().numpy(), np_bytes(rand[1:, :, ::2, 3::3]))
    with pytest.raises(ValueError):
        image_to_u8(view[:, :2])


# ------------------------------------------------------------------------------------------------------- the sampler
@torch.no_grad()
def composition(G, cr, rows, ids, step, mesh_albedo=0.6):
    """The chain from existing public pieces: decode, the kernel's cam written into the rows, render_u8, u8_to_unit, the
    generator, clamp, numpy bytes; the mesh picture from the render with an explicit 0.6 albedo and the reference's
    clamp(floor(.)/255, 0, 1) * 2 - 1 before the same bytes."""
    from gif_b200.eye_centering import eye_camera
    from gif_b200.image_decode import u8_to_unit
    n, S = rows.shape[0], cr.image_size
    verts, _ = cr.flame.decode_vertices(rows[:, :100].contiguous(), rows[:, 100:150].contiguous(), rows[:, 150:156].contiguous())
    centred = rows.clone()
    centred[:, 156:159] = eye_camera(verts)
    cond_u8 = cr.render_u8(centred)
    cond = torch.empty(n, 6, S, S, device=rows.device)
    u8_to_unit(cond_u8[:n], cond[:, 0:3])
    u8_to_unit(cond_u8[n:], cond[:, 3:6])
    img = torch.clamp(G(cond, step=step, alpha=1, input_indices=ids)[0], -1, 1)
    mesh_u8 = cr.render_vertices_u8(verts, centred[:, 156:159].contiguous(), torch.full((n, 3, 256, 256), mesh_albedo, device=rows.device),
                                    centred[:, 209:236].reshape(-1, 9, 3))[:n].cpu().numpy()
    mesh_unit = np.clip(np.floor(mesh_u8.astype(np.float32)) / np.float32(255), 0, 1) * 2 - 1
    return {"images": np_bytes(img.cpu().numpy()), "conditions": cond_u8.cpu().numpy(), "cam": centred[:, 156:159].cpu().numpy(),
            "rows": centred.cpu().numpy(), "mesh": np_bytes(mesh_unit.transpose(0, 3, 1, 2))}


@pytest.mark.parametrize("mode,res,batch", [("bf16x3", 256, 4), ("tf32", 256, 4), ("fp32", 64, 4), ("bf16x3", 512, 4)])
def test_sample_equals_composition(cuda, cr, precision, mode, res, batch):
    from gif_b200.sampler import FlameSampler
    precision(mode)
    G = generator(cuda)
    rows, ids = rows_and_ids(batch, 5, cuda)
    before = rows.clone()
    out = FlameSampler(G, cr, resolution=res, batch_size=batch).sample(rows, ids)
    assert torch.equal(rows, before)
    want = composition(G, cr, rows, ids, int(np.log2(res)) - 2)
    assert tuple(out["images"].shape) == (batch, res, res, 3) and out["images"].dtype == torch.uint8
    for k, v in want.items():
        assert np.array_equal(out[k].cpu().numpy(), v), k
    assert float(out["images"].float().std()) > 1


def test_mesh_image_with_a_visible_albedo(cuda, cr, precision):
    """At the reference's 0.6 the mesh picture is black; at a grey albedo the same path makes a visible, exact picture."""
    from gif_b200.sampler import FlameSampler
    precision("tf32")
    G = generator(cuda)
    rows, ids = rows_and_ids(4, 6, cuda)
    out = FlameSampler(G, cr, resolution=64, batch_size=4, mesh_albedo=150.0).sample(rows, ids)
    want = composition(G, cr, rows, ids, 4, mesh_albedo=150.0)["mesh"]
    assert np.array_equal(out["mesh"].cpu().numpy(), want) and 0.1 < float((want > 20).mean()) < 0.9


def assert_same(a, b):
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_graph_replay_equals_eager(cuda, cr, precision):
    from gif_b200.sampler import FlameSampler
    precision("tf32")
    G = generator(cuda, seed=2)
    rows, ids = rows_and_ids(11, 8, cuda)                  # two batches of 4 and a short one of 3
    graphs = FlameSampler(G, cr, resolution=64, batch_size=4, graphs=True)
    eager = FlameSampler(G, cr, resolution=64, batch_size=4, graphs=False)
    a, b = graphs.sample(rows, ids), eager.sample(rows, ids)
    assert_same(a, b)
    assert not torch.equal(a["images"][:4], a["images"][4:8])
    rows2, ids2 = rows_and_ids(11, 9, cuda)                # replay the captured graph on new contents
    assert_same(graphs.sample(rows2, ids2), eager.sample(rows2, ids2))
    z = torch.randn(11, 512, generator=torch.Generator().manual_seed(4)).to(cuda)     # identities given as z
    assert_same(graphs.sample(rows, z), eager.sample(rows, z))
    # the padded short batch equals the same rows sampled inside a full batch
    full = eager.sample(rows[7:11].contiguous(), ids[7:11].contiguous())
    for k in ("images", "mesh", "cam", "rows"):
        assert torch.equal(a[k][8:11], full[k][1:4]), k


@pytest.mark.parametrize("mode", ["bf16x3", "tf32"])
def test_batch_independence(cuda, cr, precision, mode):
    """Permuting the rows of a batch permutes every output bitwise: no kernel on the path mixes samples."""
    from gif_b200.sampler import FlameSampler
    precision(mode)
    G = generator(cuda, seed=3)
    rows, ids = rows_and_ids(8, 12, cuda)
    perm = torch.tensor([5, 2, 7, 0, 3, 6, 1, 4], device=cuda)
    s = FlameSampler(G, cr, resolution=256, batch_size=8, graphs=False)
    a, b = s.sample(rows, ids), s.sample(rows[perm].contiguous(), ids[perm].contiguous())
    for k in ("images", "mesh", "cam", "rows"):
        assert torch.equal(a[k][perm], b[k]), k
    assert torch.equal(a["conditions"][:8][perm], b["conditions"][:8]) and torch.equal(a["conditions"][8:][perm], b["conditions"][8:])
