"""GPU: the exact bits of the tensor-core weight-gradient kernel (bf16x3 on every shape class, tf32 on the stride-1 3x3 halo
classes) and of the stride-2 tensor-core convolution (tf32 and bf16x3; tiles of one site row and of several rows and
images), on seeded inputs.  Each result is pinned by the sha256 of its float32 bytes.

The table was recorded from the kernels these replaced, and each of them gave the same table: the weight gradient with one
big-tensor tile per kw tap instead of the halo tile (tf32 and bf16x3) and, in bf16x3, with both wgmma operands in shared
memory instead of the S operand in registers; the stride-2 convolution loading its tile one site row per TMA issue.  They
issue the same MMAs on the same values in the same order into the same accumulators as the shipped kernels.

A change that alters these bits on purpose re-records the table: ``python tests/test_tc_bits_gpu.py`` prints it."""
import hashlib
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (B, Hs, Ws, Ci, Co, k, mode)   Hs/Ws = SITE grid (output for S1/S2, input for T2)
WGRAD_CASES = [
    (3, 32, 32, 64, 128, 3, 0),       # S1 3x3 (halo tile), BLOCK_N 64, odd stage count per split
    (4, 128, 128, 128, 128, 3, 0),    # the 128 -> 128 3x3 layers of the 256^2 step (batch 4)
    (2, 16, 16, 32, 256, 3, 0),       # S1 3x3, BLOCK_N 32, two 128-row tiles
    (2, 16, 16, 64, 256, 1, 0),       # S1 1x1
    (2, 16, 16, 96, 128, 1, 0),       # S1 1x1, BLOCK_N 32
    (4, 4, 4, 64, 128, 3, 0),         # narrow images: one TMA box spans the rows (and images) of a stage
    (8, 8, 8, 32, 128, 3, 0),
    (1, 64, 64, 64, 128, 3, 1),       # S2
    (4, 4, 4, 64, 128, 3, 1),
    (1, 64, 64, 128, 128, 3, 2),      # T2
    (4, 4, 4, 128, 64, 3, 2),
    (2, 16, 16, 32, 32, 3, 0),        # STACK (Cs = 32), BLOCK_N 32
    (1, 64, 128, 64, 32, 3, 0),       # STACK (halo tile), BLOCK_N 64
    (4, 4, 4, 32, 32, 3, 0),          # STACK, narrow images
    (1, 64, 64, 64, 64, 3, 0),        # narrow (AC = 2, halo tile), Cs = 64
    (3, 8, 8, 64, 64, 3, 0),          # narrow, narrow images
    (3, 16, 16, 64, 64, 1, 0),        # narrow 1x1
    (2, 16, 32, 128, 64, 3, 1),       # narrow S2
    (1, 64, 64, 64, 32, 3, 2),        # narrow T2
    (3, 16, 16, 32, 64, 1, 0),        # narrow, Cs = 32 1x1 (the second chunk repeats the first)
    (2, 8, 8, 32, 32, 1, 0),
    (1, 32, 32, 96, 128, 3, 0),       # halo tile, BLOCK_N 32
    (1, 32, 32, 32, 32, 3, 0),        # STACK (halo tile), BLOCK_N 32
    (1, 32, 32, 32, 64, 3, 0),        # narrow (halo tile), BLOCK_N 32
]
# the stride-1 3x3 classes with images at least 32 pixels wide: the ones that take the halo tile
HALO_CASES = [c for c in WGRAD_CASES if c[6] == 0 and c[5] == 3 and c[2] >= 32]
# (B, Hi, Ci, Co): stride-2 3x3 convolutions of the discriminator, Hi -> (Hi - 3) // 2 + 1
S2_CASES = [
    (2, 257, 128, 256),     # 257^2 -> 128^2: 128 x 256 tiles of one site row
    (1, 513, 64, 128),      # 513^2 -> 256^2: 256 x 128 tiles of two rows
    (1, 257, 64, 64),       # 128 x 64 tiles of one row
    (2, 33, 512, 512),      # 16^2: 16 x 8 site boxes, split-K
    (2, 17, 512, 512),      # 8^2: 8 x 8 x 2 images per box, split-K
]
FLIPS = [(False, False), (True, True)]
PRECISIONS = ["tf32", "bf16x3"]


def grids(Hs, Ws, mode):
    if mode == 0:
        return Hs, Ws, Hs, Ws
    if mode == 1:
        return 2 * Hs + 1, 2 * Ws + 1, Hs, Ws
    return Hs, Ws, 2 * Hs + 1, 2 * Ws + 1


def _name(entry):
    kind, prec, case, flip, transposed = entry
    return f"{kind}_{prec}_" + "_".join(str(v) for v in case) + f"_f{int(flip)}_t{int(transposed)}"


ENTRIES = [("wgrad", "bf16x3", c, f, t) for c in WGRAD_CASES for f, t in FLIPS]
ENTRIES += [("wgrad", "tf32", c, f, t) for c in HALO_CASES for f, t in FLIPS]
ENTRIES += [("conv_s2", p, c, f, t) for p in PRECISIONS for c in S2_CASES for f, t in FLIPS]


def _randn(shape, seed, dev):
    import torch
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g).to(dev)


def compute(entry):
    """The float32 result of one entry, computed on cuda:0 in its precision mode."""
    from gif_b200 import ops
    from gif_b200._lib import lib
    kind, prec, case, flip, transposed = entry
    dev = "cuda:0"
    ops.set_precision(prec)
    if kind == "wgrad":
        B, Hs, Ws, Ci, Co, k, mode = case
        Hi, Wi, Ho, Wo = grids(Hs, Ws, mode)
        path = lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, 3 if prec == "bf16x3" else 0)
        assert path == (3 if prec == "bf16x3" else 2), _name(entry)
        seed = B * 77 + Hs + Ws + Ci + Co + mode + k
        x, gy = _randn((B, Hi, Wi, Ci), seed, dev), _randn((B, Ho, Wo, Co), seed + 1, dev)
        return ops._wgrad_raw(x, gy, k, mode, flip, transposed)
    B, Hi, Ci, Co = case
    Ho = ops.conv_out_size(Hi, 3, ops.S2)
    impl = 3 if prec == "bf16x3" else 0
    assert lib.gifb200_conv2d_workspace_bytes(B, Hi, Hi, Ci, Ho, Ho, Co, 3, ops.S2, int(transposed), impl) > 0, _name(entry)
    seed = B * 77 + Hi + Ci + Co
    x = _randn((B, Hi, Hi, Ci), seed, dev)
    w = _randn((9, Ci, Co) if transposed else (9, Co, Ci), seed + 1, dev) / (3.0 * Ci ** 0.5)
    return ops._conv_raw(x, w, 3, ops.S2, flip, transposed, (Ho, Ho))[0]


def digest(y):
    return hashlib.sha256(y.detach().float().contiguous().cpu().numpy().tobytes()).hexdigest()


SHA256 = {
    "wgrad_bf16x3_3_32_32_64_128_3_0_f0_t0": "51c1f345927fced3fe232f6bd4700d9ac550d3d0df5bd8e9a19a15d9ba338fa1",
    "wgrad_bf16x3_3_32_32_64_128_3_0_f1_t1": "873cfd6c3c8257a3740588b449628294d4807f16580c2572a633fc0790ae2b28",
    "wgrad_bf16x3_4_128_128_128_128_3_0_f0_t0": "5e3508bdf5913329f9fd60da6b6db3cf1affd12db340e2faeec8116abcbb5106",
    "wgrad_bf16x3_4_128_128_128_128_3_0_f1_t1": "991361b86d896870c0f515083d0ed52b4a0a83de6e4bf787e4b4b2f25e949e6a",
    "wgrad_bf16x3_2_16_16_32_256_3_0_f0_t0": "4ca172a07e615a8c13ddca4962afb6d60b26415bc7b960a4131544c0a5c812e0",
    "wgrad_bf16x3_2_16_16_32_256_3_0_f1_t1": "1d95de033a5e4b3a660bbd3ba8db70c65335d3ef3457758ec3a6d781660698a8",
    "wgrad_bf16x3_2_16_16_64_256_1_0_f0_t0": "b5fe20c1b3baa35e86287126e5a296abb9225487c2521f9f0fcbfbc8c137d882",
    "wgrad_bf16x3_2_16_16_64_256_1_0_f1_t1": "ba43622f4b6d2b27646b5a58a03f97be2b52082f955e9d668e9cd73756147cb2",
    "wgrad_bf16x3_2_16_16_96_128_1_0_f0_t0": "e3d27a1e10e304918f31694e74b0b65ca4be118e76d8d5529e5629e6a6da7275",
    "wgrad_bf16x3_2_16_16_96_128_1_0_f1_t1": "3fc4bc4db7cc6e928a646d3fb3bc2af527e3ce84fc895673c35e601ed497cb79",
    "wgrad_bf16x3_4_4_4_64_128_3_0_f0_t0": "f4fd5fe9f782ec47f7b42bfa9df2623c7b134cd7becc6f9ceaacef4d8cbe12f5",
    "wgrad_bf16x3_4_4_4_64_128_3_0_f1_t1": "c53b444f892e57e67c40f66e220844ef2f0f737bf772c889f54ed89fd90e8c6f",
    "wgrad_bf16x3_8_8_8_32_128_3_0_f0_t0": "4dfcec59be537a5cb0f32643d1fed37818382d41410775022cd4cf0727505482",
    "wgrad_bf16x3_8_8_8_32_128_3_0_f1_t1": "ade839242717337f4e6c7365afeb8381a516e6e9db1d62bb2530fe77a94fa336",
    "wgrad_bf16x3_1_64_64_64_128_3_1_f0_t0": "24ccd4888da9bbfed1c14403540d1bfc3ef39b906fc5e16e5e5b0d46b4582986",
    "wgrad_bf16x3_1_64_64_64_128_3_1_f1_t1": "4908ec485033629d68f61a8416b323eba99066f1c0575536863278085ab28dcc",
    "wgrad_bf16x3_4_4_4_64_128_3_1_f0_t0": "511899e66a93e6205a1281d43883c3ea6887d1648768ae656f0dc3e3ac50994f",
    "wgrad_bf16x3_4_4_4_64_128_3_1_f1_t1": "93035bf3ad38f53c3da5df88b606bd2fb52e938cec59b699ab5743f22187bd85",
    "wgrad_bf16x3_1_64_64_128_128_3_2_f0_t0": "d42f40e31ee91ea052e0a1cd78d8bf2ee21d8deb8d75e5ebcbb08a25631fcc14",
    "wgrad_bf16x3_1_64_64_128_128_3_2_f1_t1": "4654a40122c41184cea1bc6ae77bf83fbc9ce30997230993dd52ab322c5e624d",
    "wgrad_bf16x3_4_4_4_128_64_3_2_f0_t0": "64afb94fcebfa83c9da090df87f7c8a5a1d26b065b09e9d4358e7d31e1a6e2f9",
    "wgrad_bf16x3_4_4_4_128_64_3_2_f1_t1": "03df4b06f888f54e19e63624ce3d4913e128ec99644d5a3c64b295bb6bbaad3e",
    "wgrad_bf16x3_2_16_16_32_32_3_0_f0_t0": "9b4d2eaa8b7c8b0e1f690d4d96e39707ea9ebbf143b510bcd302d6775119eabe",
    "wgrad_bf16x3_2_16_16_32_32_3_0_f1_t1": "72041c3c7a64c187d3524c460cf029288dd44c2d76e09908965a4ca553f52ff7",
    "wgrad_bf16x3_1_64_128_64_32_3_0_f0_t0": "973b52433181394518ca00562f56f2464dc2e5577497c2f33ac9139f72c6e907",
    "wgrad_bf16x3_1_64_128_64_32_3_0_f1_t1": "b6b983fef39e35cc53f35a696d393bc5675f52a8face8046e4605d913ccd8fc1",
    "wgrad_bf16x3_4_4_4_32_32_3_0_f0_t0": "b4cfe9bb35186a5446117e1d42303546757565b3083e08e035418a2cbe3d9665",
    "wgrad_bf16x3_4_4_4_32_32_3_0_f1_t1": "264cdd50765ffbc84a4a2f7e68809cd27729f2980316c32f5f7efc0f08ac6a56",
    "wgrad_bf16x3_1_64_64_64_64_3_0_f0_t0": "0314e2dc19ce707c3e99cc957bcfbc2f11d32f025ce2449da235895b111e1e1a",
    "wgrad_bf16x3_1_64_64_64_64_3_0_f1_t1": "4654393bf2a3a1c726cab5ca63a2a6fccf06b3b03e7df11c8ca96ed8c8fe1d64",
    "wgrad_bf16x3_3_8_8_64_64_3_0_f0_t0": "4e25c8d89d1c04047fa177318b47465ac8dca58b27d389ad68755537f239bff9",
    "wgrad_bf16x3_3_8_8_64_64_3_0_f1_t1": "fcf93a31b773107be884feaa59a482b241176b3eccb2db8603bfd8da768cacfc",
    "wgrad_bf16x3_3_16_16_64_64_1_0_f0_t0": "51f9bcef1a21c043aebb8c722a5b9b44cd2a34646d1edb4e2a10d2c59414889b",
    "wgrad_bf16x3_3_16_16_64_64_1_0_f1_t1": "2e76d2c64f8a22e15afcabd897f14b5a6511ec9f7955e5bfefe200bf69059396",
    "wgrad_bf16x3_2_16_32_128_64_3_1_f0_t0": "f422f53457ff831415b2420287e002231cd64010fab937abf9a74bf355084cd6",
    "wgrad_bf16x3_2_16_32_128_64_3_1_f1_t1": "030fee668bde37c37934bb7703f022abb17660b7c265d78212ed9db08d9ebaf5",
    "wgrad_bf16x3_1_64_64_64_32_3_2_f0_t0": "2389cd184641b695d3671d6e96e96fae0a2769b2f17d4d75837ffd029eb1f9c3",
    "wgrad_bf16x3_1_64_64_64_32_3_2_f1_t1": "cd320074c8406efc4f07ba6def93acd2c66717e5331835636e68c3516da2f80b",
    "wgrad_bf16x3_3_16_16_32_64_1_0_f0_t0": "023bcb3af9e6c47cf582d71a636c00d58ece5d2f512d2b5612fb991676939380",
    "wgrad_bf16x3_3_16_16_32_64_1_0_f1_t1": "6c6a50290e73a7f43e06611f88d304136fac2247ff6f58254a30ea63167ece87",
    "wgrad_bf16x3_2_8_8_32_32_1_0_f0_t0": "4adfc7988e9566adc67deaf94f534e2e7e866c0a6c7de3904e9ff2736b529253",
    "wgrad_bf16x3_2_8_8_32_32_1_0_f1_t1": "134dc2cf4ab1a10f990e76afb73cd398af5a5cffb329e16e6f819c86f5ca5281",
    "wgrad_bf16x3_1_32_32_96_128_3_0_f0_t0": "cce46294655717c4b4a0648189473ac5ef4faa1605cb16a30e9f2501d239e2d2",
    "wgrad_bf16x3_1_32_32_96_128_3_0_f1_t1": "2bb30b5bedefc84d36ea9a8f5ae3c80669f644136eef243ed3b9e9f936652941",
    "wgrad_bf16x3_1_32_32_32_32_3_0_f0_t0": "9f73f848fe052f846b0683c450f4bf9c3987b64f4bf4df3e40b9c25384a60c8e",
    "wgrad_bf16x3_1_32_32_32_32_3_0_f1_t1": "a0a08d2a0f7932ef06d41dc9348b1db45283004e338b90480856f0b3780346c0",
    "wgrad_bf16x3_1_32_32_32_64_3_0_f0_t0": "56bf67a8da39cc3d1c922b5c82d9a6aebc77507cf8e44daf21bf1c48fdee5f4d",
    "wgrad_bf16x3_1_32_32_32_64_3_0_f1_t1": "4d1f4c85e630ba52d7f3695ca04f33f8dabe8ffd7138b3655430e771b506a850",
    "wgrad_tf32_3_32_32_64_128_3_0_f0_t0": "f0b200963f4246e1a228d18b719119da9c44fad1b0e6a201cf0d94827bb42063",
    "wgrad_tf32_3_32_32_64_128_3_0_f1_t1": "0dff8b3e88bfa8abd33f434bd1db01e3015d0423186b01f4f205954a78e41c47",
    "wgrad_tf32_4_128_128_128_128_3_0_f0_t0": "8479fb5cf969418befa47427b7d4ac5c90fead4727dd953b5fbe93acd25175d4",
    "wgrad_tf32_4_128_128_128_128_3_0_f1_t1": "86e5e6bf069a2e607f32dd35460765bcb336aa3acf0c8b431bb482f6edcb4848",
    "wgrad_tf32_1_64_128_64_32_3_0_f0_t0": "35978701236f738934ec642fc436136a698575973b11461e06df24caa2517737",
    "wgrad_tf32_1_64_128_64_32_3_0_f1_t1": "31fecf79ea581cadc74867fd65cbdef17835937fa1b1cb2b3f62329918cb3631",
    "wgrad_tf32_1_64_64_64_64_3_0_f0_t0": "77ff3434a660c2958e1652893c1c7a09ec9f4b21de4ed71310857e4141d82218",
    "wgrad_tf32_1_64_64_64_64_3_0_f1_t1": "fa7ab32c009b11edfcf5c46adc3eb630955d7f5c0a38af9b77dcfcf030057a15",
    "wgrad_tf32_1_32_32_96_128_3_0_f0_t0": "e2f4c881e6aab7ca1b6008fde06bceb32beae8f05a103a09dfadc8e255a086a6",
    "wgrad_tf32_1_32_32_96_128_3_0_f1_t1": "85acae9eb5c0678e04f6957badf64815e1dcf39ad1fb6c801bab92ee35a1c2a0",
    "wgrad_tf32_1_32_32_32_32_3_0_f0_t0": "c233285058398c39ed86fc693f418744662187794f3305f405a3cbb6bdec85a7",
    "wgrad_tf32_1_32_32_32_32_3_0_f1_t1": "a5b2835af2cf3a86b1d957d0a7f96f164696eb3de8a639752cdebaebaf16fe90",
    "wgrad_tf32_1_32_32_32_64_3_0_f0_t0": "a52757264024d22bb066f2b4b650289c2794d5944beeea714d8c573a60b8f128",
    "wgrad_tf32_1_32_32_32_64_3_0_f1_t1": "697cf744ab0e4558063b43dd7766aec5cda3de8c2d74b7bd00066f2f71f497f5",
    "conv_s2_tf32_2_257_128_256_f0_t0": "859f4e5fda53107eebecb20c847fd633cccb90e3676971cc034fe4677c96f6b7",
    "conv_s2_tf32_2_257_128_256_f1_t1": "b94ffae5d6cc947099303f37bba93568fa20d3ff34889d3d09d1db7c8054c352",
    "conv_s2_tf32_1_513_64_128_f0_t0": "80b5247175f83ed82be49df6df2c0bf2b368ef42c064c6e26b474ad68c27f97a",
    "conv_s2_tf32_1_513_64_128_f1_t1": "135c15dcc7c40e44c883e29cb9726643cbf85491282d23b95cb32c62968b9b97",
    "conv_s2_tf32_1_257_64_64_f0_t0": "05a7372cce636c500addb0a059cab718784ddcef2c8976d93b5344880f2d0ab6",
    "conv_s2_tf32_1_257_64_64_f1_t1": "1055bc55d398d9e032a239fd3af76d659830ca5068e612ff180afacb8ff5e858",
    "conv_s2_tf32_2_33_512_512_f0_t0": "7d53cb32a07eff1896662ab634fb4390c8930967bd7367180c5997c3c4c9d511",
    "conv_s2_tf32_2_33_512_512_f1_t1": "05c02d7f37d6dc2f40a29f0755cc965fe62ed80f37016510f1d58c607822a946",
    "conv_s2_tf32_2_17_512_512_f0_t0": "d5a761372b6f0f87d5d2a341e6e1cc45963ae9a50d33419e436d4ffca52a56b1",
    "conv_s2_tf32_2_17_512_512_f1_t1": "39cc185bfae7141ec5a61eaa8ee725a09f2dd628fa88d4ec74576d56391c265d",
    "conv_s2_bf16x3_2_257_128_256_f0_t0": "4469e964fe04914eba4ab5ee52c2e4a776978f71335b3386e96eebf23c4c5bcd",
    "conv_s2_bf16x3_2_257_128_256_f1_t1": "4fbe5800bc3c966abac2b96423bcf6684b92b6aaebc62779cea6b90e07059c7d",
    "conv_s2_bf16x3_1_513_64_128_f0_t0": "f4dc23f11cb1498da91702b42876cf4526ade528304ef3760a3104f57acebbd1",
    "conv_s2_bf16x3_1_513_64_128_f1_t1": "a74ffeee63c67110b057dbcd2002550d1724a8b406d76be11800c576cbf34256",
    "conv_s2_bf16x3_1_257_64_64_f0_t0": "79376ec4ecabaf790c8991559d75767c319855dae906ad969e4160708ec8b805",
    "conv_s2_bf16x3_1_257_64_64_f1_t1": "8ec8c8117d73056c686ae23fb9fa22bb428e4c4e03b47f591ca5c456e085f139",
    "conv_s2_bf16x3_2_33_512_512_f0_t0": "7bf3f0c1ade0b79aa53a24f9f64b86426e47d6cd724fe9c0cf0e98ff796bae7a",
    "conv_s2_bf16x3_2_33_512_512_f1_t1": "f5c73353e8fc7509089f89f93e5dd465a98c6fa0faf0e80880d3eb80a7151350",
    "conv_s2_bf16x3_2_17_512_512_f0_t0": "62bac90bc6dd5aba1932cceb4161c4658d7dc16c648e06bee551d8c4ef1cd646",
    "conv_s2_bf16x3_2_17_512_512_f1_t1": "8925feb155fe4fcb672e8457e4d486aa99ca48df652c0cba032b9ea4cc8c72ca",
}


@pytest.fixture
def restore_precision():
    from gif_b200 import ops
    old = ops.get_precision()
    yield
    ops.set_precision(old)


@pytest.mark.parametrize("entry", ENTRIES, ids=_name)
def test_tensor_core_bits(cuda, restore_precision, entry):
    y = compute(entry)
    a = y.cpu().numpy()
    assert np.isfinite(a).all() and np.abs(a).max() > 0, _name(entry)
    assert digest(y) == SHA256[_name(entry)], f"{_name(entry)}: the bits changed"


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    print("SHA256 = {")
    for e in ENTRIES:
        print(f'    "{_name(e)}": "{digest(compute(e))}",', flush=True)
    print("}")
