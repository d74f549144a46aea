"""Float64 functional restatement of the FID InceptionV3 feature network (my_utils/pytorch_fid/inception.py: InceptionV3
with the FID blocks FIDInceptionA / C / E_1 / E_2 on torchvision's InceptionV3 layers), in plain torch (F.conv2d,
F.batch_norm, pools) on any device, and the seeded weights the tests and the golden use.

Test infrastructure only: the product network is gif_b200/inception.py on the library's own kernels.  Keys are torchvision's
(``Mixed_5b.branch1x1.conv.weight``, ``...bn.running_var``), the layout of the FID weights file."""
import hashlib

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 0.001

# (name, Ci, Co, kh, kw) of every BasicConv2d (conv without bias + BatchNorm2d(eps=0.001) + ReLU), in module order
def _a(p, cin, pool):
    return [(f"{p}.branch1x1", cin, 64, 1, 1), (f"{p}.branch5x5_1", cin, 48, 1, 1), (f"{p}.branch5x5_2", 48, 64, 5, 5),
            (f"{p}.branch3x3dbl_1", cin, 64, 1, 1), (f"{p}.branch3x3dbl_2", 64, 96, 3, 3),
            (f"{p}.branch3x3dbl_3", 96, 96, 3, 3), (f"{p}.branch_pool", cin, pool, 1, 1)]


def _c(p, c7):
    return [(f"{p}.branch1x1", 768, 192, 1, 1), (f"{p}.branch7x7_1", 768, c7, 1, 1), (f"{p}.branch7x7_2", c7, c7, 1, 7),
            (f"{p}.branch7x7_3", c7, 192, 7, 1), (f"{p}.branch7x7dbl_1", 768, c7, 1, 1),
            (f"{p}.branch7x7dbl_2", c7, c7, 7, 1), (f"{p}.branch7x7dbl_3", c7, c7, 1, 7),
            (f"{p}.branch7x7dbl_4", c7, c7, 7, 1), (f"{p}.branch7x7dbl_5", c7, 192, 1, 7), (f"{p}.branch_pool", 768, 192, 1, 1)]


def _e(p, cin):
    return [(f"{p}.branch1x1", cin, 320, 1, 1), (f"{p}.branch3x3_1", cin, 384, 1, 1), (f"{p}.branch3x3_2a", 384, 384, 1, 3),
            (f"{p}.branch3x3_2b", 384, 384, 3, 1), (f"{p}.branch3x3dbl_1", cin, 448, 1, 1),
            (f"{p}.branch3x3dbl_2", 448, 384, 3, 3), (f"{p}.branch3x3dbl_3a", 384, 384, 1, 3),
            (f"{p}.branch3x3dbl_3b", 384, 384, 3, 1), (f"{p}.branch_pool", cin, 192, 1, 1)]


CONVS = ([("Conv2d_1a_3x3", 3, 32, 3, 3), ("Conv2d_2a_3x3", 32, 32, 3, 3), ("Conv2d_2b_3x3", 32, 64, 3, 3),
          ("Conv2d_3b_1x1", 64, 80, 1, 1), ("Conv2d_4a_3x3", 80, 192, 3, 3)]
         + _a("Mixed_5b", 192, 32) + _a("Mixed_5c", 256, 64) + _a("Mixed_5d", 288, 64)
         + [("Mixed_6a.branch3x3", 288, 384, 3, 3), ("Mixed_6a.branch3x3dbl_1", 288, 64, 1, 1),
            ("Mixed_6a.branch3x3dbl_2", 64, 96, 3, 3), ("Mixed_6a.branch3x3dbl_3", 96, 96, 3, 3)]
         + _c("Mixed_6b", 128) + _c("Mixed_6c", 160) + _c("Mixed_6d", 160) + _c("Mixed_6e", 192)
         + [("Mixed_7a.branch3x3_1", 768, 192, 1, 1), ("Mixed_7a.branch3x3_2", 192, 320, 3, 3),
            ("Mixed_7a.branch7x7x3_1", 768, 192, 1, 1), ("Mixed_7a.branch7x7x3_2", 192, 192, 1, 7),
            ("Mixed_7a.branch7x7x3_3", 192, 192, 7, 1), ("Mixed_7a.branch7x7x3_4", 192, 192, 3, 3)]
         + _e("Mixed_7b", 1280) + _e("Mixed_7c", 2048))


def seeded_state_dict(seed):
    """torchvision-layout state dict of the FID network from numpy PCG64(seed): He-scaled conv weights (std sqrt(2 / fan_in)),
    BN affine 1 + 0.1 u / 0.1 u (u uniform in [-1, 1)), running statistics 0 / 1 (calibrate them, see the golden recipe), a
    zero fc layer.  float64."""
    rng = np.random.Generator(np.random.PCG64(seed))
    sd = {}
    for name, ci, co, kh, kw in CONVS:
        sd[f"{name}.conv.weight"] = torch.from_numpy(rng.standard_normal((co, ci, kh, kw)) * np.sqrt(2.0 / (ci * kh * kw)))
        sd[f"{name}.bn.weight"] = torch.from_numpy(1.0 + 0.1 * rng.uniform(-1.0, 1.0, co))
        sd[f"{name}.bn.bias"] = torch.from_numpy(0.1 * rng.uniform(-1.0, 1.0, co))
        sd[f"{name}.bn.running_mean"] = torch.zeros(co, dtype=torch.float64)
        sd[f"{name}.bn.running_var"] = torch.ones(co, dtype=torch.float64)
        sd[f"{name}.bn.num_batches_tracked"] = torch.zeros((), dtype=torch.long)
    sd["fc.weight"] = torch.zeros(1008, 2048, dtype=torch.float64)
    sd["fc.bias"] = torch.zeros(1008, dtype=torch.float64)
    return sd


def weights_sha256(sd):
    """sha256 of the conv weights (float64 bytes, CONVS order): pins the generator."""
    h = hashlib.sha256()
    for name, *_ in CONVS:
        h.update(sd[f"{name}.conv.weight"].double().contiguous().numpy().tobytes())
    return h.hexdigest()


def _conv(sd, name, x, stride=1, padding=0):
    t = lambda k: sd[f"{name}.{k}"].to(x)
    y = F.conv2d(x, t("conv.weight"), stride=stride, padding=padding)
    y = F.batch_norm(y, t("bn.running_mean"), t("bn.running_var"), t("bn.weight"), t("bn.bias"), False, 0.0, BN_EPS)
    return F.relu(y)


def _avg(x):
    return F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)


def _mixed_a(sd, p, x):
    b1 = _conv(sd, f"{p}.branch1x1", x)
    b5 = _conv(sd, f"{p}.branch5x5_2", _conv(sd, f"{p}.branch5x5_1", x), padding=2)
    b3 = _conv(sd, f"{p}.branch3x3dbl_1", x)
    b3 = _conv(sd, f"{p}.branch3x3dbl_3", _conv(sd, f"{p}.branch3x3dbl_2", b3, padding=1), padding=1)
    return torch.cat([b1, b5, b3, _conv(sd, f"{p}.branch_pool", _avg(x))], 1)


def _mixed_b(sd, p, x):
    b3 = _conv(sd, f"{p}.branch3x3", x, stride=2)
    bd = _conv(sd, f"{p}.branch3x3dbl_2", _conv(sd, f"{p}.branch3x3dbl_1", x), padding=1)
    bd = _conv(sd, f"{p}.branch3x3dbl_3", bd, stride=2)
    return torch.cat([b3, bd, F.max_pool2d(x, 3, 2)], 1)


def _mixed_c(sd, p, x):
    b1 = _conv(sd, f"{p}.branch1x1", x)
    b7 = _conv(sd, f"{p}.branch7x7_1", x)
    b7 = _conv(sd, f"{p}.branch7x7_2", b7, padding=(0, 3))
    b7 = _conv(sd, f"{p}.branch7x7_3", b7, padding=(3, 0))
    bd = _conv(sd, f"{p}.branch7x7dbl_1", x)
    for i, pad in ((2, (3, 0)), (3, (0, 3)), (4, (3, 0)), (5, (0, 3))):
        bd = _conv(sd, f"{p}.branch7x7dbl_{i}", bd, padding=pad)
    return torch.cat([b1, b7, bd, _conv(sd, f"{p}.branch_pool", _avg(x))], 1)


def _mixed_d(sd, p, x):
    b3 = _conv(sd, f"{p}.branch3x3_2", _conv(sd, f"{p}.branch3x3_1", x), stride=2)
    b7 = _conv(sd, f"{p}.branch7x7x3_1", x)
    b7 = _conv(sd, f"{p}.branch7x7x3_2", b7, padding=(0, 3))
    b7 = _conv(sd, f"{p}.branch7x7x3_3", b7, padding=(3, 0))
    b7 = _conv(sd, f"{p}.branch7x7x3_4", b7, stride=2)
    return torch.cat([b3, b7, F.max_pool2d(x, 3, 2)], 1)


def _mixed_e(sd, p, x, max_pool):
    b1 = _conv(sd, f"{p}.branch1x1", x)
    b3 = _conv(sd, f"{p}.branch3x3_1", x)
    b3 = torch.cat([_conv(sd, f"{p}.branch3x3_2a", b3, padding=(0, 1)), _conv(sd, f"{p}.branch3x3_2b", b3, padding=(1, 0))], 1)
    bd = _conv(sd, f"{p}.branch3x3dbl_2", _conv(sd, f"{p}.branch3x3dbl_1", x), padding=1)
    bd = torch.cat([_conv(sd, f"{p}.branch3x3dbl_3a", bd, padding=(0, 1)),
                    _conv(sd, f"{p}.branch3x3dbl_3b", bd, padding=(1, 0))], 1)
    pool = F.max_pool2d(x, 3, 1, 1) if max_pool else _avg(x)
    return torch.cat([b1, b3, bd, _conv(sd, f"{p}.branch_pool", pool)], 1)


def forward(sd, inp, output_blocks=(3,), resize_input=True, normalize_input=True):
    """InceptionV3.forward (inception.py:130-164): inp (B,3,H,W) in [0,1] -> list of the requested blocks' NCHW maps.
    Computed in inp's dtype and device (float64 for the golden)."""
    x = inp
    if resize_input:
        x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False)
    if normalize_input:
        x = 2 * x - 1
    blocks = [
        lambda x: F.max_pool2d(_conv(sd, "Conv2d_2b_3x3", _conv(sd, "Conv2d_2a_3x3", _conv(sd, "Conv2d_1a_3x3", x, stride=2)),
                                     padding=1), 3, 2),
        lambda x: F.max_pool2d(_conv(sd, "Conv2d_4a_3x3", _conv(sd, "Conv2d_3b_1x1", x)), 3, 2),
        lambda x: _block2(sd, x),
        lambda x: F.adaptive_avg_pool2d(_mixed_e(sd, "Mixed_7c", _mixed_e(sd, "Mixed_7b", _mixed_d(sd, "Mixed_7a", x), False),
                                                 True), (1, 1)),
    ]
    out = []
    for i, blk in enumerate(blocks[:max(output_blocks) + 1]):
        x = blk(x)
        if i in output_blocks:
            out.append(x)
    return out


def _block2(sd, x):
    x = _mixed_a(sd, "Mixed_5b", x)
    x = _mixed_a(sd, "Mixed_5c", x)
    x = _mixed_a(sd, "Mixed_5d", x)
    x = _mixed_b(sd, "Mixed_6a", x)
    for p in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        x = _mixed_c(sd, p, x)
    return x


def golden_state_dict(g):
    """The golden's weights: seeded_state_dict(seed) with the calibrated BN running statistics stored in the golden ``g``."""
    sd = seeded_state_dict(int(g["seed"]))
    for name, *_ in CONVS:
        sd[f"{name}.bn.running_mean"] = torch.from_numpy(g[f"bn_mean/{name}"])
        sd[f"{name}.bn.running_var"] = torch.from_numpy(g[f"bn_var/{name}"])
    return sd


def golden_inputs(g):
    """(name, images in [0,1] (float64), resize_input) of the golden cases, regenerated from their seeds."""
    out = []
    for name, shape, seed, resize in (("299", (2, 3, 299, 299), 31, True), ("256", (2, 3, 256, 256), 32, True),
                                      ("256_noresize", (2, 3, 256, 256), 33, False)):
        x = torch.from_numpy(np.random.Generator(np.random.PCG64(seed)).uniform(0.0, 1.0, shape))
        out.append((name, x, resize))
    return out
