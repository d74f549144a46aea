"""TEST INFRASTRUCTURE ONLY -- writes ``tests/golden/fid_real.npz``: the real-image FID statistics of a seeded PNG folder as
the UNMODIFIED reference computes them (my_utils/pytorch_fid/fid_score.py ``calculate_activation_statistics``, the call
of my_utils/compute_fid.py:43-45 with ``cuda=False``), on the CPU.

  * Network: the reference InceptionV3 with the weights of ``tests/golden/fid_inception.npz`` (seeded conv / BN affine
    weights, calibrated BN statistics: ``inception_oracle.golden_state_dict``), loaded as ``tools/make_fid_golden.py`` does:
    the torch hub loaders are replaced by a function that raises before the module is imported, and the module's own
    loader name is pointed at the state dict.
  * Folder: ``synth_images.png_folder(dir, 70, 512, SEED)`` (1/f spectrum, written by Pillow), so that 64 images are used
    and the remainder of 6 is dropped.  The PNG byte stream depends on the zlib build, the pixels do not: the sha256 of
    every decoded image is stored and the tests check the folder they regenerate against it.
  * Statistics at resolution 256 for dims 192 and 2048, by the reference's function on the reference network in float64
    (its float32 batch, v / 255, widened exactly): ``mu`` and ``sigma`` in full for 192, ``mu`` and seeded samples of
    ``sigma`` (``golden_util.sample``) plus its float64 sum for 2048.  The same function on the float32 network gives
    the reference's own float32 error (``ref32_err_*``), stored beside them.

Run where the reference tree and torchvision exist (a few minutes on 8 cores):   python tools/make_fid_real_golden.py
"""
import copy
import hashlib
import os
import sys
import tempfile

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import golden_util as gu  # noqa: E402
from gif_b200.synth_images import png_folder  # noqa: E402
from make_fid_golden import _as_blocks, load_reference_fid_module, rel_l2  # noqa: E402
from oracle import inception_oracle as IO  # noqa: E402
from oracle import ref_import  # noqa: E402

SEED = 4000
N_FILES, SIZE, RESOLUTION = 70, 512, 256
SIGMA_SAMPLES, SIGMA_SAMPLE_SEED = 8192, 7


def pixel_sha256(path):
    return hashlib.sha256(np.ascontiguousarray(np.array(Image.open(path))).tobytes()).hexdigest()


class _Float64(torch.nn.Module):
    """The float64 reference network behind the float32 batch the reference's get_activations builds."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        return self.net(x.double())


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    ref = load_reference_fid_module()
    import my_utils.pytorch_fid.fid_score as fid_score
    sd = IO.golden_state_dict(gu.load_golden("fid_inception.npz"))
    ref.load_state_dict_from_url = lambda *a, **k: sd
    out = {"seed": np.int64(SEED), "n_files": np.int64(N_FILES), "size": np.int64(SIZE),
           "resolution": np.int64(RESOLUTION), "weights_sha256": np.array(IO.weights_sha256(sd))}
    with tempfile.TemporaryDirectory() as d:
        files = png_folder(d, N_FILES, SIZE, SEED)
        out["pixel_sha256"] = np.array([pixel_sha256(f) for f in files])
        for dims in (192, 2048):
            with ref_import.quiet():
                net32 = ref.InceptionV3([ref.InceptionV3.BLOCK_INDEX_BY_DIM[dims]])
            net64 = copy.deepcopy(net32).double()
            missing, _ = net64.load_state_dict(_as_blocks(sd), strict=False)   # the float64 values, later blocks dropped
            assert not [k for k in missing if not k.endswith("num_batches_tracked")], missing
            with ref_import.quiet():
                mu, sigma = fid_score.calculate_activation_statistics(sorted(files), _Float64(net64), 32, dims, cuda=False,
                                                                      resolution=RESOLUTION)
                mu32, sigma32 = fid_score.calculate_activation_statistics(sorted(files), net32, 32, dims, cuda=False,
                                                                          resolution=RESOLUTION)
            out[f"ref32_err_mu_{dims}"] = rel_l2(mu32, mu)
            out[f"ref32_err_sigma_{dims}"] = rel_l2(sigma32, sigma)
            out[f"mu_{dims}"] = mu
            if dims == 192:
                out["sigma_192"] = sigma
            else:
                out["sigma_2048"], out["sigma_2048_sum"] = gu.sample(torch.from_numpy(sigma), SIGMA_SAMPLES, SIGMA_SAMPLE_SEED)
            print(dims, "done: reference float32 error mu", out[f"ref32_err_mu_{dims}"], "sigma",
                  out[f"ref32_err_sigma_{dims}"], flush=True)
    np.savez_compressed(os.path.join(gu.GOLDEN_DIR, "fid_real.npz"), **{k: np.asarray(v) for k, v in out.items()})
    print("written", os.path.join(gu.GOLDEN_DIR, "fid_real.npz"))


if __name__ == "__main__":
    main()
