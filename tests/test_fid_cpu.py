"""Evaluation path (SURVEY 8f.4): Frechet distance and streaming activation statistics against the reference's formulas
(my_utils/pytorch_fid/fid_score.py:142-196 = scipy sqrtm of the covariance product; compute_fid.py:79-80 = np.mean / np.cov),
and against the stored result of the reference's own function."""
import numpy as np
import pytest
import torch
from scipy import linalg

from gif_b200 import fid


def _ref_frechet(mu1, sigma1, mu2, sigma2):
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    return diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean.real)


@pytest.mark.parametrize("d,n", [(8, 50), (64, 200), (256, 300)])
def test_frechet_distance_matches_sqrtm_form(d, n):
    rng = np.random.default_rng(d)
    a, b = rng.normal(size=(n, d)), rng.normal(size=(n, d)) * 1.3 + 0.2
    m1, s1, m2, s2 = a.mean(0), np.cov(a, rowvar=False), b.mean(0), np.cov(b, rowvar=False)
    got = fid.calculate_frechet_distance(m1, s1, m2, s2, device=torch.device("cpu"))
    want = _ref_frechet(m1, s1, m2, s2)
    assert abs(got - want) < 1e-7 * max(1.0, abs(want))
    assert abs(fid.calculate_frechet_distance(m1, s1, m1, s1, device=torch.device("cpu"))) < 1e-8 * d


def test_frechet_distance_matches_reference_function_live():
    """The reference's own calculate_frechet_distance (fid_score.py:142-196) on seeded statistics; its result is stored in
    tests/golden/reference_live.npz (oracle/make_live_golden.py)."""
    import golden_util as gu
    import live_cases
    want = float(gu.load_golden("reference_live.npz")["fid_reference"][0])
    m1, s1, m2, s2 = live_cases.fid_case()
    assert abs(fid.calculate_frechet_distance(m1, s1, m2, s2, device=torch.device("cpu")) - want) < 1e-7 * abs(want)


def test_streaming_statistics_and_fid_computer(tmp_path):
    class Feat(torch.nn.Module):                                # stand-in with pytorch_fid.InceptionV3's interface
        def __init__(self):
            super().__init__()
            self.conv = torch.nn.Conv2d(3, 16, 3, stride=2)

        def forward(self, x):
            return [torch.tanh(self.conv(x))]
    torch.manual_seed(0)
    model = Feat()
    imgs = torch.rand(70, 3, 16, 16) * 2 - 1                     # generator output range
    fc = fid.FidComputer(true_img_stats_dir=str(tmp_path), model=model, dims=16, device=torch.device("cpu"))
    mu, cov = fc.compute_sats_given_img_tensor(imgs.clone())
    x = imgs - imgs.min()
    x = x / x.max()                                              # compute_fid.py:53-55
    with torch.no_grad():
        feats = torch.nn.functional.adaptive_avg_pool2d(model(x)[0], 1).reshape(70, -1).double().numpy()
    assert np.allclose(mu.numpy(), feats.mean(0), atol=1e-12) and np.allclose(cov.numpy(), np.cov(feats, rowvar=False), atol=1e-12)
    np.savez(tmp_path / "ffhq_16X16_fid_stats.npz", mu=feats.mean(0) + 0.1, sigma=np.cov(feats, rowvar=False) * 1.5)
    want = _ref_frechet(feats.mean(0) + 0.1, np.cov(feats, rowvar=False) * 1.5, feats.mean(0), np.cov(feats, rowvar=False))
    assert abs(fc.get_fid(imgs.clone()) - want) < 1e-8 * max(1.0, abs(want))
    u8 = (x * 255).to(torch.uint8)
    fc.compute_sats_given_img_tensor(u8)                         # uint8 path (compute_fid.py:56-57)
    with pytest.raises(ValueError):
        fc.compute_sats_given_img_tensor(imgs.double())
