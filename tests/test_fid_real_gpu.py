"""GPU: the real images' FID statistics computed on the device (gif_b200/fid_real.py).

  (a) ``gifb200_resize_bilinear_u8`` is bitwise ``gifb200_resize_bilinear`` of the float batch v / 255 (numpy's IEEE
      division), and ``InceptionV3`` on a uint8 batch is bitwise ``InceptionV3`` on that float batch;
  (b) the device decode + resize of a seeded PNG folder is bitwise ``np.array(Image.open(f).resize((R, R)))``;
  (c) mu / sigma against ``tests/golden/fid_real.npz`` (the unmodified reference's ``calculate_activation_statistics``
      on the CPU in float64, tools/make_fid_real_golden.py), with the bars of tests/test_fid_inception_gpu.py: fp32 2e-5,
      bf16x3 2e-4, each scaled by the reference's own float32 error on the quantity over its float32 error on the
      network's 256^2 features (as that test scales its bars); tf32 printed only;
  (d) ``FidComputer`` computes and caches the statistics, and a second computer reproduces the FID bit for bit from the
      cache alone;
  (e) two passes give bitwise-equal statistics."""
import hashlib
import os
import shutil

import numpy as np
import pytest
import torch
from PIL import Image

import golden_util as gu
from gif_b200 import fid_real, ops
from gif_b200.fid import FidComputer
from gif_b200.inception import InceptionV3
from gif_b200.synth_images import noise, photo, png_folder
from oracle import inception_oracle as IO

pytestmark = pytest.mark.gpu

BARS = {"fp32": 2e-5, "bf16x3": 2e-4}


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.fixture(scope="module")
def golden():
    return gu.load_golden("fid_real.npz")


@pytest.fixture(scope="module")
def inception_golden():
    return gu.load_golden("fid_inception.npz")


@pytest.fixture(scope="module")
def sd(inception_golden):
    return IO.golden_state_dict(inception_golden)


@pytest.fixture(scope="module")
def folder(tmp_path_factory, golden):
    """The golden's seeded folder, regenerated; its pixels are checked against the golden's hashes."""
    d = tmp_path_factory.mktemp("fid_real_pngs")
    files = png_folder(d, int(golden["n_files"]), int(golden["size"]), int(golden["seed"]))
    got = [hashlib.sha256(np.ascontiguousarray(np.array(Image.open(f))).tobytes()).hexdigest() for f in files]
    assert got == [str(h) for h in golden["pixel_sha256"]], "the regenerated folder's pixels differ from the golden's"
    return str(d)


@pytest.fixture()
def precision(request):
    old = ops.get_precision()
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(old)


def _u8_cases():
    rng = np.random.default_rng(5)
    ramp = np.arange(256 * 256 * 3, dtype=np.int64).reshape(256, 256, 3) % 256       # every byte value
    cases = {"256": np.stack([ramp, np.asarray(photo(256, 256, 1)), np.asarray(noise(256, 256, 2))]).astype(np.uint8),
             "1024": np.stack([np.asarray(photo(1024, 1024, 3)), np.asarray(noise(1024, 1024, 4))]),
             "299": np.stack([np.asarray(photo(299, 299, 5)), np.asarray(noise(299, 299, 6))]),
             "37x53": rng.integers(0, 256, (3, 37, 53, 3), dtype=np.uint8)}
    return cases


@pytest.mark.parametrize("round_tf32", [0, 1])
@pytest.mark.parametrize("case", ["256", "1024", "299", "37x53", "strided"])
def test_resize_u8_bitwise_equals_float_kernel(cuda, case, round_tf32):
    cases = _u8_cases()
    if case == "strided":                                   # every other image of a batch: batch stride 2*H*W*3
        base = np.concatenate([cases["256"], cases["256"][::-1]])
        x_np = base[::2]
        x = torch.from_numpy(base).to(cuda)[::2]
        assert x.stride(0) == 2 * 256 * 256 * 3
    else:
        x_np = cases[case]
        x = torch.from_numpy(x_np).to(cuda)
    f = torch.from_numpy(x_np.astype(np.float32) / np.float32(255)).to(cuda).permute(0, 3, 1, 2)    # numpy's IEEE division
    for size, scale, shift in (((299, 299), 2.0, -1.0), ((299, 299), 1.0, 0.0)):
        want = ops.resize_bilinear(f, size, 32, scale, shift, round_tf32=bool(round_tf32))
        got = ops.resize_bilinear_u8(x, size, 32, scale, shift, round_tf32=bool(round_tf32))
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (case, scale, int((got != want).sum()))


def test_inception_uint8_input_bitwise(cuda, sd):
    x_np = _u8_cases()["256"]
    net = InceptionV3([1, 3], weights=sd).to(cuda)
    with torch.no_grad():
        got = net(torch.from_numpy(x_np).to(cuda))
        want = net(torch.from_numpy(x_np.astype(np.float32) / np.float32(255)).to(cuda).permute(0, 3, 1, 2))
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@pytest.mark.parametrize("R", [256, 299])
def test_device_decode_and_resize_bitwise_pillow(cuda, tmp_path, R):
    if R == 256:                                             # mixed sizes: resized, already R^2 (not resized), odd sizes
        files = [str(tmp_path / f"{i}.png") for i in range(5)]
        for f, (h, w, s) in zip(files, [(512, 512, 1), (256, 256, 2), (300, 200, 3), (512, 512, 4), (97, 311, 5)]):
            photo(h, w, s).save(f)
    else:
        files = png_folder(tmp_path, 4, 512, 9)
    status = torch.zeros(len(files), dtype=torch.int32, device=cuda)
    x = fid_real.device_batch(files, [fid_real.load_png(f) for f in files], R, status, cuda).cpu().numpy()
    assert (status.cpu() == 0).all()
    for f, got in zip(files, x):
        img = Image.open(f)
        want = np.array(img.resize((R, R)) if R != 299 else img)
        assert np.array_equal(got, want), f


def test_size_mismatch_at_299_raises(cuda, tmp_path):
    files = [str(tmp_path / "a.png"), str(tmp_path / "b.png")]
    photo(64, 64, 1).save(files[0])
    photo(64, 80, 2).save(files[1])
    with pytest.raises(ValueError, match="b.png"):
        fid_real.device_batch(files, [fid_real.load_png(f) for f in files], 299, torch.zeros(2, dtype=torch.int32,
                                                                                                device=cuda), cuda)


def test_decode_of_the_golden_folder_bitwise_pillow(cuda, folder, golden):
    R = int(golden["resolution"])
    files = fid_real.real_image_files(folder)[:8]
    status = torch.zeros(len(files), dtype=torch.int32, device=cuda)
    x = fid_real.device_batch(files, [fid_real.load_png(f) for f in files], R, status, cuda).cpu().numpy()
    for f, got in zip(files, x):
        assert np.array_equal(got, np.array(Image.open(f).resize((R, R)))), f


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "tf32"], indirect=True)
def test_statistics_against_reference_golden(cuda, folder, golden, inception_golden, sd, precision):
    R = int(golden["resolution"])
    floor = float(inception_golden["256_ref32_err"])
    failures = []
    for dims in (192, 2048):
        net = InceptionV3([InceptionV3.BLOCK_INDEX_BY_DIM[dims]], weights=sd).to(cuda)
        mu, sigma = fid_real.real_image_statistics(folder, R, net, dims)
        mu, sigma = mu.cpu().numpy(), sigma.cpu()
        e_mu = rel_l2(mu, golden[f"mu_{dims}"])
        if dims == 192:
            e_sigma = rel_l2(sigma.numpy(), golden["sigma_192"])
        else:
            samp, total = gu.sample(sigma, golden["sigma_2048"].size, 7)
            e_sigma = rel_l2(samp, golden["sigma_2048"])
            e_sum = abs(total - float(golden["sigma_2048_sum"])) / float(sigma.abs().sum())    # the whole matrix, loosely
            print(f"{precision} dims 2048: sigma sum error {e_sum:.2e} of sum |sigma|")
            if precision != "tf32" and not e_sum < BARS[precision]:
                failures.append((dims, "sigma sum", e_sum, BARS[precision]))
        print(f"{precision} dims {dims}: mu rel L2 {e_mu:.2e} (reference fp32 {float(golden[f'ref32_err_mu_{dims}']):.2e}), "
              f"sigma {e_sigma:.2e} (reference fp32 {float(golden[f'ref32_err_sigma_{dims}']):.2e})")
        if precision == "tf32":
            continue
        for name, e in (("mu", e_mu), ("sigma", e_sigma)):
            bar = BARS[precision] * max(1.0, float(golden[f"ref32_err_{name}_{dims}"]) / floor)
            if not e < bar:
                failures.append((dims, name, e, bar))
    assert not failures, failures


def test_fid_computer_computes_caches_and_reuses(cuda, tmp_path, folder, sd):
    src = tmp_path / "imgs"
    shutil.copytree(folder, src)
    stats_dir = tmp_path / "stats"
    images = gu.rand_uniform((64, 3, 256, 256), 91)
    fc = FidComputer(database_root_dir=str(src), true_img_stats_dir=str(stats_dir), inception_weights=sd, device=cuda)
    fid1 = fc.get_fid(images)
    path = stats_dir / "ffhq_256X256_fid_stats.npz"
    assert os.listdir(stats_dir) == [path.name]
    with np.load(path) as f:
        assert f["mu"].shape == (2048,) and f["sigma"].shape == (2048, 2048) and f["sigma"].dtype == np.float64
        assert np.array_equal(f["mu"][:], fc.m_t) and np.array_equal(f["sigma"][:], fc.s_t)
    shutil.rmtree(src)
    fc2 = FidComputer(database_root_dir=str(src), true_img_stats_dir=str(stats_dir), inception_weights=sd, device=cuda)
    fid2 = fc2.get_fid(images)
    print(f"FID {fid1!r} / from the cache {fid2!r}")
    assert fid1 == fid2 and np.isfinite(fid1)


def test_statistics_deterministic(cuda, folder, sd):
    net = InceptionV3([3], weights=sd).to(cuda)
    a = fid_real.real_image_statistics(folder, 256, net, 2048, threads=3)
    b = fid_real.real_image_statistics(folder, 256, net, 2048, threads=8)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
