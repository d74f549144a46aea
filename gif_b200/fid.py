"""Evaluation loop, second half (SURVEY 8f.4): FID of the EMA generator's images -- ``my_utils/compute_fid.py`` (FidComputer,
:10-87) and ``my_utils/pytorch_fid/fid_score.py`` (compute_activation_batch :126-139, calculate_frechet_distance :142-196),
same class / method names and return values, with the statistics kept ON THE DEVICE:

  * activations are reduced as they are produced -- a float64 running sum and a running sum of outer products (2048 x 2048) --
    instead of a (10 000, 2048) host array followed by ``np.mean`` / ``np.cov`` (compute_fid.py:66-82): no device->host copy per
    batch, same unbiased estimator;
  * the Frechet distance uses the symmetric form Tr sqrt(C1 C2) = sum sqrt(eig(C1^1/2 C2 C1^1/2)) (two ``eigh`` calls in
    float64, on the device when there is one) instead of scipy's Schur-based ``sqrtm`` of the non-symmetric product
    (fid_score.py:176): same value for positive semi-definite covariances, no complex round trip.

The feature extractor is the FID Inception network of pytorch_fid (torchvision's InceptionV3 with the FID weights,
pt_inception-2015-12-05).  ``FidComputer(inception_weights=...)`` builds ``gif_b200.inception.InceptionV3`` -- the network on
this library's own kernels (general-geometry convolution, pooling, bilinear resize), forward only, in the precision of
``ops.set_precision`` -- from a weights path or state dict (``inception_weights=True``: the standard file under
$TORCH_HOME; it is never downloaded).  A model can still be INJECTED instead (any module mapping (B,3,H,W) in [0,1] to a list
whose first element is (B,C,h,w) features, which is the interface of pytorch_fid.InceptionV3).  The generator side of the
loop is gif_b200/inference.py."""
import os

import numpy as np
import torch
import torch.nn.functional as F


def _psd_sqrt(c):
    w, v = torch.linalg.eigh(c)
    return (v * w.clamp_min(0).sqrt()) @ v.transpose(-1, -2)


def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6, device=None):
    """fid_score.py:142-196.  Accepts numpy arrays or tensors; computed in float64."""
    dev = device or (torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu"))
    t = lambda a: torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a, dtype=torch.float64, device=dev)
    mu1, mu2, s1, s2 = t(mu1).reshape(-1), t(mu2).reshape(-1), torch.atleast_2d(t(sigma1)), torch.atleast_2d(t(sigma2))
    if mu1.shape != mu2.shape:
        raise ValueError("Training and test mean vectors have different lengths")
    if s1.shape != s2.shape:
        raise ValueError("Training and test covariances have different dimensions")
    diff = mu1 - mu2
    a = _psd_sqrt(s1)
    lam = torch.linalg.eigvalsh(a @ s2 @ a)
    if not torch.isfinite(lam).all():                         # fid_score.py:177-182: regularise a singular product
        off = torch.eye(s1.shape[0], dtype=torch.float64, device=dev) * eps
        a = _psd_sqrt(s1 + off)
        lam = torch.linalg.eigvalsh(a @ (s2 + off) @ a)
    tr_covmean = lam.clamp_min(0).sqrt().sum()
    return float(diff.dot(diff) + torch.trace(s1) + torch.trace(s2) - 2 * tr_covmean)


class ActivationStatistics:
    """Streaming mean / unbiased covariance (np.mean(axis=0), np.cov(rowvar=False)) of feature rows, float64, on the device."""

    def __init__(self, dims, device):
        self.n = 0
        self.s = torch.zeros(dims, dtype=torch.float64, device=device)
        self.ss = torch.zeros(dims, dims, dtype=torch.float64, device=device)

    def update(self, feats):
        f = feats.reshape(feats.shape[0], -1).to(torch.float64)
        self.n += f.shape[0]
        self.s += f.sum(0)
        self.ss += f.t() @ f

    def finalize(self):
        mu = self.s / self.n
        cov = (self.ss - self.n * torch.outer(mu, mu)) / (self.n - 1)
        return mu, cov


def compute_activation_batch(model, batch):
    """fid_score.py:126-139, result left on the device."""
    pred = model(batch)[0]
    if pred.shape[2] != 1 or pred.shape[3] != 1:
        pred = F.adaptive_avg_pool2d(pred, output_size=(1, 1))
    return pred.reshape(batch.shape[0], -1)


class FidComputer:
    """compute_fid.py:10-87.  ``model``: the FID Inception network, or None with ``inception_weights`` to build the native one
    for ``dims`` (see the module docstring); ``true_img_stats_dir`` holds the reference's ``ffhq_{R}X{R}_fid_stats.npz`` files
    (mu, sigma), computed from the PNGs in ``database_root_dir`` when missing (``compute_true_img_response``)."""

    def __init__(self, database_root_dir=None, true_img_stats_dir=None, model=None, dims=2048, device=None,
                 inception_weights=None):
        if model is None:
            if inception_weights is None:
                raise ValueError("FidComputer needs the FID Inception network: pass model=... (e.g. pytorch_fid.InceptionV3) "
                                 "or inception_weights=<path or state dict> (True: search $TORCH_HOME)")
            from .inception import InceptionV3
            model = InceptionV3([InceptionV3.BLOCK_INDEX_BY_DIM[dims]],
                                weights=None if inception_weights is True else inception_weights)
        self.dims = dims
        self.true_data_loc = database_root_dir
        self.true_img_stats_dir = true_img_stats_dir
        self.device = device or (torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu"))
        self.model = model.to(self.device).eval()
        self.m_t, self.s_t = None, None
        self.current_resolution = None

    def compute_true_img_response(self, resolution):
        """compute_fid.py:26-46: the statistics of the real images at this resolution.  Loaded from
        ``true_img_stats_dir/ffhq_{R}X{R}_fid_stats.npz`` when it exists; otherwise computed from ``database_root_dir/*.png``
        with this computer's network (``fid_real.real_image_statistics``: sorted file names, the reference's selection and
        resize rules) and, when ``true_img_stats_dir`` is set, written there atomically for the next run."""
        path = os.path.join(self.true_img_stats_dir or "", f"ffhq_{resolution}X{resolution}_fid_stats.npz")
        if os.path.exists(path):
            with np.load(path) as f:
                self.m_t, self.s_t = f["mu"][:], f["sigma"][:]
            return
        if self.true_data_loc is None:
            raise FileNotFoundError(f"{path}: statistics of the real images not found, and no image folder "
                                    "(database_root_dir) to compute them from")
        from .fid_real import real_image_statistics, save_statistics
        mu, sigma = real_image_statistics(self.true_data_loc, resolution, self.model, self.dims, device=self.device)
        self.m_t, self.s_t = mu.cpu().numpy(), sigma.cpu().numpy()
        if self.true_img_stats_dir is not None:
            save_statistics(path, self.m_t, self.s_t)

    def compute_sats_given_img_tensor(self, imag_tensor, batch_size=32):
        """compute_fid.py:48-82: float32 images are range-normalised to [0,1] over the WHOLE tensor, uint8 divided by 255."""
        t = imag_tensor if torch.is_tensor(imag_tensor) else torch.from_numpy(np.asarray(imag_tensor))
        if t.dtype == torch.float32:
            lo = t.min()
            scale = (t - lo).max()
            prep = lambda b: (b.to(self.device, non_blocking=True) - lo.to(self.device)) / scale.to(self.device)
        elif t.dtype == torch.uint8:
            prep = lambda b: b.to(self.device, non_blocking=True).float() / 255
        else:
            raise ValueError("Datatype of Image tensor not undestood: " + str(t.dtype))
        stats = ActivationStatistics(self.dims, self.device)
        with torch.no_grad():
            for i in range(0, t.shape[0], batch_size):
                stats.update(compute_activation_batch(self.model, prep(t[i:i + batch_size])))
        return stats.finalize()

    def get_fid(self, imag_tensor):
        resolution = imag_tensor.shape[-1]
        if self.m_t is None or self.current_resolution != resolution:
            self.compute_true_img_response(resolution)
            self.current_resolution = resolution
        m2, s2 = self.compute_sats_given_img_tensor(imag_tensor)
        return calculate_frechet_distance(self.m_t, self.s_t, m2, s2, device=self.device)
