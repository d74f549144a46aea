"""CPU: host logic of the 512^2 / 1024^2 configurations -- the weight-gradient path and workspace queries for the narrow
(64- and 32-channel) layers, their one-wave grids, the unchanged queries of the shapes that were on the tensor cores
before, and the dataset's host-side resize of 256^2 renders to 512^2 images."""
import io

import numpy as np
import torch

from gif_b200 import data

SMS = 132

# (B, Hi, Wi, Ci, Ho, Wo, Co, k, mode): the layers of a 512^2 / 1024^2 G+D step whose small side has 32 or 64 channels
NARROW = [
    (16, 512, 512, 64, 512, 512, 64, 3, 0),      # G progression.7.st_cv2; D ResBlock(64->128).conv1 @512
    (16, 512, 512, 32, 512, 512, 64, 3, 0),      # G noise conv 24->64 (input padded to 32)
    (4, 512, 512, 64, 1025, 1025, 32, 3, 2),     # G progression.8.st_cv1 (upsampling, T2)
    (16, 512, 512, 32, 512, 512, 64, 1, 0),      # D 512 stem 9->64 (input padded to 32)
    (4, 1024, 1024, 32, 1024, 1024, 32, 1, 0),   # D 1024 stem 9->32
    (4, 1025, 1025, 32, 512, 512, 64, 3, 1),     # D 1024 ResBlock(32->64).conv2 (S2)
    (4, 512, 512, 32, 512, 512, 64, 1, 0),       # D 1024 ResBlock(32->64).skip
    (3, 8, 8, 128, 8, 8, 64, 3, 0),              # Cb = 128
    (3, 4, 8, 64, 4, 8, 32, 1, 0),               # Cs = 32, Cb = 64
]

# (B, H, Ci, Co, mode) -> wgrad workspace bytes and split count of the shapes already on the tensor cores
EXISTING = {
    (32, 256, 128, 128, 0): (12976384, 22), (32, 128, 256, 256, 0): (11796736, 5), (32, 64, 512, 512, 0): (9437440, 1),
    (32, 32, 512, 512, 0): (9437440, 1), (32, 257, 128, 256, 1): (12976384, 11), (32, 129, 256, 512, 1): (9437440, 2),
    (32, 128, 256, 128, 2): (12976384, 11), (32, 64, 512, 256, 2): (9437440, 2), (16, 256, 128, 128, 0): (12976384, 22),
    (8, 64, 512, 512, 0): (9437440, 1),
}


def test_narrow_wgrad_queries_and_one_wave():
    from gif_b200._lib import lib
    for (B, Hi, Wi, Ci, Ho, Wo, Co, k, mode) in NARROW:
        args = (B, Hi, Wi, Ci, Ho, Wo, Co, k, mode)
        for impl in (0, 2, 3):
            assert lib.gifb200_conv2d_wgrad_path(*args, impl) == (3 if impl == 3 else 2), (args, impl)
        assert lib.gifb200_conv2d_wgrad_path(*args, 1) == 1
        ws = lib.gifb200_conv2d_wgrad_workspace_bytes(*args, 0)
        splits = (ws - 256) // (k * k * Co * Ci * 4)
        assert ws == splits * k * k * Co * Ci * 4 + 256, args
        small, big = (Ci, Co) if mode == 2 else (Co, Ci)
        ctas = (big // (64 if big % 64 == 0 else 32)) * k * splits        # one 64-row tile covers the small side
        assert small in (32, 64) and 1 <= splits and ctas <= SMS, (args, splits, ctas)
        units = B * (Hi * Wi if mode == 2 else Ho * Wo) // 32                 # 32-pixel units of the small grid
        assert ctas > SMS // 2 or splits == units, (args, splits, ctas)      # the split count fills the wave


def test_existing_wgrad_queries_unchanged():
    from gif_b200._lib import lib
    for (B, H, Ci, Co, mode), (ws_want, splits_want) in EXISTING.items():
        Ho = H if mode == 0 else ((H - 3) // 2 + 1 if mode == 1 else 2 * H + 1)
        assert lib.gifb200_conv2d_wgrad_path(B, H, H, Ci, Ho, Ho, Co, 3, mode, 0) == 2
        assert lib.gifb200_conv2d_wgrad_path(B, H, H, Ci, Ho, Ho, Co, 3, mode, 3) == 3
        ws = lib.gifb200_conv2d_wgrad_workspace_bytes(B, H, H, Ci, Ho, Ho, Co, 3, mode, 0)
        assert ws == ws_want and (ws - 256) // (9 * Co * Ci * 4) == splits_want, (B, H, Ci, Co, mode, ws)


def test_narrow_shapes_outside_the_variant_stay_on_simt():
    from gif_b200._lib import lib
    assert lib.gifb200_conv2d_wgrad_path(4, 33, 33, 64, 16, 16, 32, 3, 1, 0) == 1      # Cs = 32, S2
    assert lib.gifb200_conv2d_wgrad_path(4, 16, 16, 32, 33, 33, 64, 3, 2, 0) == 1      # Cs = 32, T2
    assert lib.gifb200_conv2d_wgrad_path(4, 16, 16, 48, 16, 16, 64, 3, 0, 0) == 1      # Cb = 48 (not a multiple of 32)
    assert lib.gifb200_conv2d_wgrad_path(4, 16, 16, 32, 16, 16, 96, 3, 0, 0) == 1      # Cs = 96
    assert lib.gifb200_conv2d_wgrad_workspace_bytes(4, 16, 16, 32, 16, 16, 96, 3, 0, 0) == 0
    # Cs = 32 (1x1) with 128 big channels: the R1 term of the 256^2 discriminator stem keeps the exact kernel and its bits
    assert lib.gifb200_conv2d_wgrad_path(32, 256, 256, 128, 256, 256, 32, 1, 0, 0) == 1


def _png(arr):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(arr).save(b, format="PNG")
    return b.getvalue()


def test_dataset_512_images_with_256_renders(tmp_path):
    """resolution=512, rend_flm_res=256: the 256^2 renders and normal maps are resized to 512^2 on the host."""
    from PIL import Image
    n, R, r = 4, 512, 256
    rng = np.random.default_rng(1)
    imgs = rng.integers(0, 256, (n, R, R, 3), dtype=np.uint8)
    rend = rng.integers(0, 256, (n, r, r, 3), dtype=np.uint8)
    nrm = rng.integers(0, 256, (n, r, r, 3), dtype=np.uint8)
    data.write_lmdb(str(tmp_path / "real"), [(data.image_key(R, i), _png(imgs[i])) for i in range(n)] + [(b"length", str(n).encode())])
    data.write_lmdb(str(tmp_path / "rend"), [(data.image_key(r, i), _png(rend[i])) for i in range(n)] +
                    [(data.normal_map_key(r, i), _png(nrm[i])) for i in range(n)])
    ds = data.GifLmdbDataset(str(tmp_path / "real"), str(tmp_path / "rend"), np.zeros((n, 159), np.float32), resolution=R,
                             rend_flm_res=r)
    img, cond, _, idx = ds[2]
    assert idx == 2 and tuple(img.shape) == (3, R, R) and tuple(cond[0].shape) == (6, R, R)
    want = np.asarray(Image.fromarray(rend[2]).resize((R, R)), np.float32)
    assert torch.allclose(cond[0][:3], torch.from_numpy(want).permute(2, 0, 1) / 255.0 * 2 - 1, atol=1e-6)
