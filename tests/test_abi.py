"""CPU: the C-ABI library loads, exports every symbol include/gifb200.h declares, the ctypes table matches the header's
argument counts, shape errors are reported through return codes (no compute calls: there is no GPU here), and the
drop-in modules keep the reference's state_dict layout."""
import ctypes
import os
import re

import pytest
import torch

import golden_util as gu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "gifb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(?:int|size_t|long long|const char\*)\s+(gifb200_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S):
        args = m.group(2).strip()
        n = 0 if args in ("", "void") else len([a for a in args.split(",") if a.strip()])
        out[m.group(1)] = n
    return out


def test_library_exports_header():
    from gif_b200 import _lib
    fns = header_functions()
    assert len(fns) >= 23
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name, nargs in fns.items():
        assert hasattr(lib, name), f"{name} declared in gifb200.h but not exported"
        assert name in _lib.SIGNATURES, f"{name} missing from the ctypes table"
        assert len(_lib.SIGNATURES[name][1]) == nargs, f"{name}: ctypes table has wrong arity"
    assert set(_lib.SIGNATURES) == set(fns)
    assert _lib.lib.gifb200_version() >= 100


def test_error_codes_without_gpu():
    from gif_b200 import _lib
    rc = _lib.lib.gifb200_upfirdn2d(None, None, None, 1, 4, 4, 4, 4, 4, 9, 9, 1, 1, 0, 0, 0, 0, None)
    assert rc == -1 and b"8x8" in _lib.lib.gifb200_last_error()
    rc = _lib.lib.gifb200_conv2d(None, None, None, 1, 8, 8, 4, 8, 8, 4, 5, 0, 0, 0, 1, 0, None, 1.0, 1.0, 0, None, 0, None)
    assert rc == -1
    assert _lib.lib.gifb200_rasterize_workspace_bytes(2, 100, 64, 64) > 0


def test_dispatch_queries_and_one_wave_split_count():
    """Host logic that needs no GPU: which path a shape takes, workspace sizes, and that the weight-gradient kernel's grid
    (128-channel tiles x kernel rows x pixel splits, ONE CTA per SM) never exceeds the 132 SMs of an H100 SXM -- a second
    wave of a few straggler CTAs doubles that kernel's time."""
    from gif_b200 import _lib
    lib = _lib.lib
    bn = lambda c: 64 if c % 64 == 0 else 32
    for (B, H, Ci, Co, mode) in [(32, 256, 128, 128, 0), (32, 128, 256, 256, 0), (32, 64, 512, 512, 0), (32, 32, 512, 512, 0),
                                 (32, 257, 128, 256, 1), (32, 129, 256, 512, 1), (32, 128, 256, 128, 2), (32, 64, 512, 256, 2),
                                 (16, 256, 128, 128, 0), (8, 64, 512, 512, 0)]:
        Ho = H if mode == 0 else ((H - 3) // 2 + 1 if mode == 1 else 2 * H + 1)
        assert lib.gifb200_conv2d_workspace_bytes(B, H, H, Ci, Ho, Ho, Co, 3, mode, 0, 0) >= 9 * Co * Ci * 4   # staged weights
        assert lib.gifb200_conv2d_wgrad_path(B, H, H, Ci, Ho, Ho, Co, 3, mode, 0) == 2
        wws = lib.gifb200_conv2d_wgrad_workspace_bytes(B, H, H, Ci, Ho, Ho, Co, 3, mode, 0)
        splits = wws // (9 * Co * Ci * 4)
        small, big = (Ci, Co) if mode == 2 else (Co, Ci)
        ctas = (small // 128) * (big // bn(big)) * 3 * splits
        assert 1 <= splits and 96 <= ctas <= 132, (B, H, Ci, Co, mode, splits, ctas)
    # shapes outside the tensor-core path: exact fp32 kernels, no workspace
    assert lib.gifb200_conv2d_wgrad_path(32, 256, 256, 9, 256, 256, 128, 3, 0, 0) == 1
    assert lib.gifb200_conv2d_wgrad_path(32, 256, 256, 9, 256, 256, 128, 3, 0, 2) == 0        # forcing the tensor-core path is refused
    assert lib.gifb200_conv2d_workspace_bytes(32, 250, 250, 128, 250, 250, 128, 3, 0, 0, 0) == 0   # ragged size -> SIMT
    assert lib.gifb200_flame_lbs_workspace_bytes(64, 5) == 64 * (36 + 60) * 4
    rc = lib.gifb200_flame_lbs(None, None, None, None, None, None, None, None, None, None, None, 4, 5023, 150, 9, None, 0, None)
    assert rc == -1 and b"joints" in lib.gifb200_last_error()
    rc = lib.gifb200_texture_steal_fwd(None, None, None, None, None, None, None, None, None, 1, 0, 8, 3, 10, 256, None)
    assert rc == -1 and b"texture_steal" in lib.gifb200_last_error()


def test_state_dict_layout_matches_reference_manifest():
    from gif_b200.model.stg2_discriminator import Discriminator
    from gif_b200.model.stg2_generator import StyledGenerator
    G = StyledGenerator(embedding_vocab_size=100, rendered_flame_ascondition=True, normal_maps_as_cond=True)
    want = gu.g_shapes(100)
    got = {k: tuple(v.shape) for k, v in G.state_dict().items()}
    assert list(got) == list(want) and got == {k: tuple(v) for k, v in want.items()}
    assert sum(p.numel() for p in G.parameters()) == 31_633_991          # SURVEY M1 [probe]
    for size in (64, 256):
        D = Discriminator(size, num_color_chnls=9)
        want = gu.d_shapes(size)
        got = {k: tuple(v.shape) for k, v in D.state_dict().items()}
        assert list(got) == list(want) and got == {k: tuple(v) for k, v in want.items()}
    assert sum(p.numel() for p in D.parameters()) == 28_864_897          # SURVEY M2 [probe]
    # a reference-style checkpoint (seeded) loads strictly
    G.load_state_dict(gu.seeded_state_dict(gu.g_shapes(100), 1), strict=True)


def test_no_cpu_fallback():
    from gif_b200 import ops
    from gif_b200._lib import GifB200Error
    with pytest.raises(GifB200Error):
        ops.conv2d(torch.zeros(1, 4, 4, 8), torch.zeros(9, 8, 8), 3)
    with pytest.raises(GifB200Error):
        ops.upfirdn2d(torch.zeros(1, 4, 4, 8), gu.blur_kernel())


def test_install_as_reference_modules():
    import gif_b200
    gif_b200.install_as_reference_modules(data_parallel=False)
    import model.stg2_generator as g
    import model.stylegan2_common_layers as cl
    assert hasattr(g, "StyledGenerator") and hasattr(cl, "ModulatedConv2d") and hasattr(cl, "upfirdn2d")


def test_discriminator_construction_and_minibatch_stddev_glue():
    """CPU-checkable parts of the discriminator module: layer widths / key layout for every size, and the minibatch
    standard-deviation feature against the oracle's restatement of disc.py:59-65."""
    import torch
    from gif_b200.model.stg2_discriminator import Discriminator, _channel_table, minibatch_stddev_feature
    from oracle import stylegan2_oracle as O
    assert _channel_table(2) == {4: 512, 8: 512, 16: 512, 32: 512, 64: 512, 128: 256, 256: 128, 512: 64, 1024: 32}
    assert _channel_table(1)[64] == 256 and _channel_table(1)[1024] == 16
    for size, nblocks in ((4, 0), (16, 2), (256, 6), (1024, 8)):
        D = Discriminator(size, num_color_chnls=9)
        assert len(D.convs) == 1 + nblocks
        assert D.convs[0][0].weight.shape == (_channel_table(2)[size], 9, 1, 1)
        assert D.final_conv[0].weight.shape == (512, 513, 3, 3) and D.final_linear[0].weight.shape == (512, 8192)
    g = torch.Generator().manual_seed(0)
    for b in (1, 3, 4, 8, 32):
        x = torch.randn(b, 512, 4, 4, generator=g, dtype=torch.float64)
        if b % min(b, 4) != 0:
            continue
        y = minibatch_stddev_feature(x)
        assert y.shape == (b, 513, 4, 4) and torch.equal(y[:, :512], x)
        assert (y - O.minibatch_stddev(x, 4)).abs().max() < 1e-14
