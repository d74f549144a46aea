"""CPU: the FID Inception oracle against the golden of the unmodified reference network, weight loading (both key layouts,
strict keys, no download), BatchNorm folding, FidComputer's construction rules and the workspace queries of the new
convolution entry point."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu
from oracle import inception_oracle as IO


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.fixture(scope="module")
def golden():
    return gu.load_golden("fid_inception.npz")


def test_oracle_matches_golden(golden):
    sd = IO.golden_state_dict(golden)
    assert IO.weights_sha256(sd) == str(golden["weights_sha256"]), "seeded weight generator drifted"
    for case, x, resize in IO.golden_inputs(golden)[1:]:          # the 256^2 cases (resize and map sizes 127..6)
        out = IO.forward(sd, x, (0, 1, 2, 3), resize_input=resize)
        assert rel_l2(out[3].reshape(2, -1).numpy(), golden[f"{case}_b3"]) < 1e-12
        for i in range(3):
            assert tuple(out[i].shape) == tuple(golden[f"{case}_b{i}_shape"])
            assert rel_l2(gu.sample(out[i], 4096, 40 + i)[0], golden[f"{case}_b{i}"]) < 1e-12


def _blocks_layout(sd):
    from gif_b200.inception import BLOCKS
    out = {}
    for bi, mods in enumerate(BLOCKS):
        for j, (mod, _) in enumerate(mods):
            for k, v in sd.items():
                if k.startswith(mod + "."):
                    out[f"blocks.{bi}.{j}" + k[len(mod):]] = v
    return out


def test_weight_layouts_and_strict_keys():
    from gif_b200.inception import canonical_state_dict
    sd = IO.seeded_state_dict(1)
    a = canonical_state_dict(sd)                                  # torchvision names, fc.* and num_batches_tracked ignored
    b = canonical_state_dict(_blocks_layout(sd))                  # pytorch_fid's InceptionV3.state_dict() names
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert len(a) == 94 * 5
    with pytest.raises(KeyError, match="unexpected"):
        canonical_state_dict({**sd, "Mixed_5b.branch9x9.conv.weight": torch.zeros(1)})
    with pytest.raises(KeyError, match="unexpected"):
        canonical_state_dict({**sd, "AuxLogits.fc.weight": torch.zeros(1)})
    bad = dict(sd)
    del bad["Mixed_7c.branch_pool.bn.running_var"]
    with pytest.raises(KeyError, match="missing"):
        canonical_state_dict(bad)
    assert len(canonical_state_dict(bad, blocks=range(3))) < len(a)   # a network up to block 2 does not need it


def test_bn_folding_matches_batchnorm_eval():
    from gif_b200.inception import BN_EPS, fold_bn
    g = torch.Generator().manual_seed(0)
    conv = torch.nn.Conv2d(48, 64, (1, 7), padding=(0, 3), bias=False).double()
    bn = torch.nn.BatchNorm2d(64, eps=BN_EPS).double().eval()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g, dtype=torch.float64))
        bn.weight.copy_(torch.rand(64, generator=g, dtype=torch.float64) + 0.5)
        bn.bias.copy_(torch.randn(64, generator=g, dtype=torch.float64))
        bn.running_mean.copy_(torch.randn(64, generator=g, dtype=torch.float64))
        bn.running_var.copy_(torch.rand(64, generator=g, dtype=torch.float64) + 0.1)
    x = torch.randn(2, 48, 9, 11, generator=g, dtype=torch.float64)
    w, b = fold_bn(conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var)
    with torch.no_grad():
        want = bn(conv(x))
    got = F.conv2d(x, w, b, padding=(0, 3))
    assert float((got - want).abs().max() / want.abs().max()) < 1e-14


def test_missing_weights_file_never_downloads(monkeypatch, tmp_path):
    import torch.hub
    import urllib.request
    from gif_b200 import inception

    def boom(*a, **k):
        raise AssertionError("a download function was called")

    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", boom)
    monkeypatch.setattr(torch.hub, "download_url_to_file", boom)
    monkeypatch.setattr(urllib.request, "urlopen", boom)
    monkeypatch.setattr(urllib.request, "urlretrieve", boom)
    monkeypatch.setenv("TORCH_HOME", str(tmp_path))
    with pytest.raises(FileNotFoundError) as e:
        inception.InceptionV3()
    assert str(tmp_path / inception.FID_WEIGHTS_FILE) in str(e.value)
    assert str(tmp_path / "hub" / "checkpoints" / inception.FID_WEIGHTS_FILE) in str(e.value)
    with pytest.raises(FileNotFoundError):
        inception.InceptionV3(weights=str(tmp_path / "nothing.pth"))


def test_weights_file_hash_and_weights_only_load(tmp_path, monkeypatch):
    from gif_b200 import inception
    sd = {k: v.float() for k, v in IO.seeded_state_dict(3).items()}
    bad = tmp_path / "hub" / "checkpoints" / inception.FID_WEIGHTS_FILE
    bad.parent.mkdir(parents=True)
    torch.save(sd, bad)
    monkeypatch.setenv("TORCH_HOME", str(tmp_path))
    with pytest.raises(RuntimeError, match="sha256"):             # the seeded file does not carry the real hash prefix
        inception.InceptionV3()
    good = tmp_path / "fid_seeded.pth"                            # no hash in the name: loaded as is (weights_only)
    torch.save(sd, good)
    net = inception.InceptionV3(output_blocks=[1], weights=str(good))
    assert set(net.convs) == {"Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3", "Conv2d_3b_1x1", "Conv2d_4a_3x3"}
    assert net.convs["Conv2d_3b_1x1"].weight.shape == (1, 96, 64)          # 80 output channels padded to 96
    assert net.convs["Conv2d_1a_3x3"].weight.shape == (9, 32, 32)          # 3 input channels padded to 32
    assert net.state_dict() == {}
    with pytest.raises(NotImplementedError):
        inception.InceptionV3(use_fid_inception=False, weights=sd)


def test_fid_computer_construction():
    from gif_b200.fid import FidComputer
    with pytest.raises(ValueError):
        FidComputer(model=None)
    fc = FidComputer(dims=192, inception_weights=IO.seeded_state_dict(4), device=torch.device("cpu"))
    assert fc.model.output_blocks == [1] and fc.model.last_needed_block == 1
    injected = torch.nn.Identity()
    assert FidComputer(model=injected, device=torch.device("cpu")).model is injected


def test_conv_ex_workspace_queries_on_cpu():
    from gif_b200 import _lib
    from gif_b200.inception import BLOCKS
    lib = _lib.lib
    convs = [c for mods in BLOCKS for _, cs in mods for c in cs]
    assert len(convs) == 94
    assert len({(c[1], c[2], c[3], c[4], c[5], c[6], c[7]) for c in convs}) == 43
    for name, ci, co, kh, kw, s, ph, pw in convs:
        ci, co = (ci + 31) // 32 * 32, (co + 31) // 32 * 32
        for B in (2, 33):
            H = 35
            Ho, Wo = (H + 2 * ph - kh) // s + 1, (H + 2 * pw - kw) // s + 1
            n = lib.gifb200_conv2d_ex_workspace_bytes(B, H, H, ci, Ho, Wo, co, kh, kw, s, ph, pw, 2)
            assert n >= kh * kw * ci * co * 4, name
            assert lib.gifb200_conv2d_ex_workspace_bytes(B, H, H, ci, Ho, Wo, co, kh, kw, s, ph, pw, 1) == 0
    # outside the tensor-core path: no workspace (exact fp32 SIMT kernel)
    assert lib.gifb200_conv2d_ex_workspace_bytes(2, 35, 35, 3, 35, 35, 32, 3, 3, 1, 1, 1, 0) == 0
    # split-K partials for a small 8x8 layer
    small = lib.gifb200_conv2d_ex_workspace_bytes(2, 8, 8, 448, 8, 8, 384, 3, 3, 1, 1, 1, 2)
    assert small > 9 * 448 * 384 * 4 + 2 * 64 * 384 * 4
    # geometry errors are return codes
    rc = lib.gifb200_conv2d_ex(None, None, None, 1, 8, 8, 32, 8, 8, 32, 9, 9, 1, 4, 4, 32, 0, 1, 0, None, 0, None, 0, None)
    assert rc == -1 and b"geometry" in lib.gifb200_last_error()
    rc = lib.gifb200_pool2d(None, None, 1, 8, 8, 4, 3, 3, 3, 0, 0, 4, 0, 0, None)
    assert rc == -1
