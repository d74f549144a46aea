"""GPU: gif_b200.inception.InceptionV3 (the FID feature network on the library's kernels) against the golden of the unmodified
reference network in every precision mode, against the float64 oracle evaluated live on the device at 1024^2, a profiler
check that no library convolution or pooling kernel runs, and FID of seeded-generator images with native features against
FID with oracle features.

Bars on block 3 (relative L2): fp32 2e-5, bf16x3 2e-4, tf32 5e-3; blocks 0-2 (seeded samples) use the same bars.  They hold
as they are on the 256^2 resize case and on 1024^2 inputs.  The seeded network amplifies float32 rounding about 60x through
block 2 on the 299^2 and the un-resized 256^2 inputs: there the reference's OWN float32 error is 9-12x that of the 256^2 case
(3.1e-5 / 4.0e-5 vs 3.4e-6, tests/golden/FID_ORACLE_VS_REFERENCE.txt), and the bars are scaled by that ratio.  tf32 (10-bit
operands) does not reach its scaled bar on those two cases (4.7e-2 measured on the 299^2 case, H100): its error is printed,
not asserted.  FID of two sets of seeded-generator images is small (8.2 at 2048 dims, 6.5e-5 at 192): fp32 holds 1e-3
(measured 5e-5 / 1e-4), bf16x3 is asserted at 1e-2 (measured 3.2e-3), tf32 is printed only (its features move FID by
several times its value here)."""
import numpy as np
import pytest
import torch

import golden_util as gu
from gif_b200 import ops
from gif_b200.fid import ActivationStatistics, FidComputer, calculate_frechet_distance
from gif_b200.inception import InceptionV3
from oracle import inception_oracle as IO

pytestmark = pytest.mark.gpu

BARS = {"fp32": 2e-5, "bf16x3": 2e-4, "tf32": 5e-3}


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


@pytest.fixture(scope="module")
def golden():
    return gu.load_golden("fid_inception.npz")


@pytest.fixture(scope="module")
def sd(golden):
    return IO.golden_state_dict(golden)


@pytest.fixture()
def precision(request):
    old = ops.get_precision()
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(old)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "tf32"], indirect=True)
def test_blocks_against_golden(cuda, golden, sd, precision):
    nets = {r: InceptionV3([0, 1, 2, 3], resize_input=r, weights=sd).to(cuda) for r in (True, False)}
    floor = float(golden["256_ref32_err"])
    failures = []
    for case, x, resize in IO.golden_inputs(golden):
        scale = max(1.0, float(golden[f"{case}_ref32_err"]) / floor)
        with torch.no_grad():
            out = nets[resize](x.float().to(cuda))
        e3 = rel_l2(out[3].reshape(2, -1).cpu().numpy(), golden[f"{case}_b3"])
        errs = [rel_l2(gu.sample(out[i], 4096, 40 + i)[0], golden[f"{case}_b{i}"]) for i in range(3)]
        print(f"{precision} {case}: block 3 rel L2 {e3:.2e}, blocks 0-2 {', '.join(f'{e:.2e}' for e in errs)}")
        for i in range(3):
            assert tuple(out[i].shape) == tuple(golden[f"{case}_b{i}_shape"])
        if precision == "tf32" and scale > 1.0:
            continue
        if not (e3 < BARS[precision] * scale and max(errs) < BARS[precision] * scale):
            failures.append((case, scale, e3, errs))
    assert not failures, failures


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "tf32"], indirect=True)
def test_1024_against_live_oracle(cuda, sd, precision):
    x = torch.from_numpy(np.random.Generator(np.random.PCG64(77)).uniform(0.0, 1.0, (2, 3, 1024, 1024)))
    sd_dev = {k: v.to(cuda) for k, v in sd.items()}
    with torch.no_grad():
        want = IO.forward(sd_dev, x.to(cuda), (3,))[0]
        got = InceptionV3([3], weights=sd).to(cuda)(x.float().to(cuda).contiguous(memory_format=torch.channels_last))[0]
    e = rel_l2(got.reshape(2, -1).cpu().numpy(), want.reshape(2, -1).cpu().numpy())
    print(f"{precision} 1024^2: block 3 rel L2 {e:.2e}")
    assert e < BARS[precision]


def test_no_library_convolution_or_pooling(cuda, sd):
    net = InceptionV3([0, 1, 2, 3], weights=sd).to(cuda)
    x = torch.rand(4, 3, 256, 256, device=cuda)
    with torch.no_grad():
        net(x)                                            # warm-up (staging)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                torch.profiler.ProfilerActivity.CUDA]) as prof:
            net(x)
            torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    bad_ops = [n for n in names if n.startswith("aten::") and any(s in n for s in ("conv", "cudnn", "pool", "upsample",
                                                                                    "interpolate", "mkldnn"))]
    assert not bad_ops, sorted(set(bad_ops))
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("conv_ex_tc_kernel" in n for n in kernels)
    foreign = [n for n in kernels if "gifb200" not in n and any(s in n.lower() for s in ("conv", "cudnn", "pool", "xmma",
                                                                                           "implicit", "upsample"))]
    assert not foreign, sorted(set(foreign))


@pytest.fixture(scope="module")
def generator_images(cuda):
    """1024 images of the seeded 256^2 generator: two sets of 512 (from different conditions)."""
    from gif_b200.inference import get_images_from_flame_params
    from gif_b200.model.stg2_generator import StyledGenerator
    G = StyledGenerator(embedding_vocab_size=16, rendered_flame_ascondition=True, normal_maps_as_cond=True)
    G.load_state_dict(gu.seeded_state_dict(gu.g_shapes(16), 5))
    G.to(cuda)
    old = ops.get_precision()
    ops.set_precision("bf16x3")
    try:
        sets = []
        for seed in (61, 62):
            cond = gu.rand_uniform((512, 6, 256, 256), seed)
            idx = gu.randint(16, (512,), seed + 10)
            with torch.no_grad():
                sets.append(get_images_from_flame_params(cond, None, G, step=6, alpha=1, input_indices=idx, batch_size=32,
                                                         device=cuda))
    finally:
        ops.set_precision(old)
    return sets


def _oracle_stats(sd_dev, images, blocks, cuda):
    lo, scale = images.min(), (images - images.min()).max()      # FidComputer's range normalisation of float32 images
    stats = {b: ActivationStatistics(d, cuda) for b, d in blocks.items()}
    with torch.no_grad():
        for i in range(0, images.shape[0], 32):
            batch = ((images[i:i + 32].to(cuda) - lo.to(cuda)) / scale.to(cuda)).double()
            outs = IO.forward(sd_dev, batch, tuple(sorted(blocks)))
            for b, o in zip(sorted(blocks), outs):
                stats[b].update(torch.nn.functional.adaptive_avg_pool2d(o, (1, 1)).reshape(o.shape[0], -1))
    return {b: s.finalize() for b, s in stats.items()}


@pytest.fixture(scope="module")
def oracle_fid_stats(cuda, sd, generator_images):
    sd_dev = {k: v.to(cuda) for k, v in sd.items()}
    return [_oracle_stats(sd_dev, imgs, {1: 192, 3: 2048}, cuda) for imgs in generator_images]


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "tf32"], indirect=True)
@pytest.mark.parametrize("dims", [2048, 192])
def test_fid_native_vs_oracle_features(cuda, sd, generator_images, oracle_fid_stats, precision, dims):
    block = InceptionV3.BLOCK_INDEX_BY_DIM[dims]
    (m_t, s_t), (m_o, s_o) = oracle_fid_stats[0][block], oracle_fid_stats[1][block]
    fc = FidComputer(dims=dims, inception_weights=sd, device=cuda)
    fc.m_t, fc.s_t, fc.current_resolution = m_t, s_t, 256
    fid_native = fc.get_fid(generator_images[1])
    fid_oracle = calculate_frechet_distance(m_t, s_t, m_o, s_o, device=cuda)
    e = abs(fid_native - fid_oracle) / abs(fid_oracle)
    print(f"{precision} dims {dims}: FID native {fid_native:.6f} oracle {fid_oracle:.6f} rel diff {e:.2e}")
    if precision != "tf32":
        assert e < (1e-3 if precision == "fp32" else 1e-2)
