"""GPU: the training iteration at 512^2 and 1024^2 (batch 4, R1, with and without the texture-interpolation loss, whose
256^2 condition reaches the generator through the upsampling pyramid): eager and CUDA-graph iterations agree, parameters
stay finite, and no SIMT convolution or weight-gradient kernel runs in the tensor-core modes."""
import pytest
import torch

import golden_util as gu

pytestmark = pytest.mark.gpu


def _batch(seed, b, res, dev):
    return (gu.rand_uniform((b, 3, res, res), seed).to(dev), gu.rand_uniform((b, 6, res, res), seed + 1).to(dev),
            gu.randint(16, (b,), seed + 2).to(dev))


def _flame(b, dev):
    g = torch.Generator().manual_seed(2)
    return torch.cat([torch.randn(b, 150, generator=g), (torch.rand(b, 6, generator=g) * 2 - 1) * 0.3,
                      torch.rand(b, 1, generator=g) * 3 + 7, (torch.rand(b, 2, generator=g) * 2 - 1) * 0.02], 1).to(dev)


@pytest.mark.parametrize("texture", [False, True])
@pytest.mark.parametrize("res", [512, 1024])
def test_highres_eager_and_graph_iterations_agree(cuda, tf32_mode, res, texture):
    """As test_trainer_gpu.py: d_loss depends only on the weights at the start of the iteration and is compared tightly;
    g_loss comes after D's Adam step (a sign-like update that amplifies summation-order noise) and is compared loosely.
    The texture term draws its interpolation weight, pairs and identity from the device RNG inside the step; the RNG is
    reseeded before each trainer's iteration so that both draw the same values."""
    from gif_b200.train_step import GifTrainer
    b = 4
    kw = dict(vocab=16, r1_every=2, ppl=False, seed=3, texture_loss=b if texture else False)
    t_e, t_g = GifTrainer(cuda, res, **kw), GifTrainer(cuda, res, **kw)
    extra = (_flame(b, cuda),) if texture else ()

    def both(it):
        t_e.generator.load_state_dict(t_g.generator.state_dict())
        t_e.discriminator.load_state_dict(t_g.discriminator.state_dict())
        torch.cuda.manual_seed(100 + it)      # both trainers draw the same texture-term randoms
        oe = [float(v) for v in t_e.train_iteration(*_batch(10 * it, b, res, cuda), *extra)]
        torch.cuda.manual_seed(100 + it)
        og = [float(v) for v in t_g.train_iteration(*_batch(10 * it, b, res, cuda), *extra)]
        assert all(v == v and abs(v) < 1e4 for v in oe + og), (oe, og)
        assert oe[0] == pytest.approx(og[0], rel=2e-4, abs=1e-5), (it, oe, og)
        assert oe[1] == pytest.approx(og[1], rel=5e-2, abs=1e-3), (it, oe, og)

    for it in range(2):
        both(it)
    t_g.capture(b, res)
    assert t_g._graphs is not None and t_g.graph_launches[True] > t_g.graph_launches[False] > 100
    for it in range(2, 4):       # both R1 variants from the graphs
        both(it)
    torch.cuda.synchronize()
    assert all(torch.isfinite(p).all() for p in t_g.generator.parameters())
    assert all(torch.isfinite(p).all() for p in t_g.discriminator.parameters())


@pytest.mark.parametrize("precision", ["tf32", "bf16x3"])
@pytest.mark.parametrize("res", [512, 1024])
def test_highres_step_runs_no_simt_kernels(cuda, res, precision):
    """The bench.py step (R1, path-length term): no SIMT convolution, and the only SIMT weight gradient is the R1 term of
    the 4x4 final_conv (513 channels padded to 544), which runs on SIMT at every resolution, 256^2 included.  The
    texture-interpolation term is left out: its generator pass runs on B - 1 interpolated labels, and at B = 4 the 4x4
    layer's 3 * 16 pixels are not a multiple of the weight-gradient kernel's 32-pixel unit, at every resolution."""
    from torch.profiler import ProfilerActivity, profile

    from gif_b200 import ops
    from gif_b200._lib import lib
    from gif_b200.train_step import GifTrainer
    old = ops.get_precision()
    ops.set_precision(precision)
    try:
        b = 4
        tr = GifTrainer(cuda, res, vocab=16, r1_every=2, ppl=True, seed=4)
        tr.train_iteration(*_batch(0, b, res, cuda))
        torch.cuda.synchronize()
        ops.PROFILE = []           # every weight-gradient launch records its shape
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for it in (1, 2):    # iteration 2 carries R1
                tr.train_iteration(*_batch(10 * it, b, res, cuda))
            torch.cuda.synchronize()
        shapes = [e[-1] for e in ops.PROFILE]
    finally:
        ops.PROFILE = None
        ops.set_precision(old)
    names = {e.name for e in prof.events() if e.device_type.name == "CUDA"}
    assert any("wgrad_tc_kernel" in n for n in names)
    assert not any("conv_simt_kernel" in n for n in names)
    simt = set()
    for kind, mode, B, Hi, Wi, Ci, Co, k in shapes:
        Ho, Wo = ops.conv_out_size(Hi, k, mode), ops.conv_out_size(Wi, k, mode)
        if kind == "wgrad" and lib.gifb200_conv2d_wgrad_path(B, Hi, Wi, Ci, Ho, Wo, Co, k, mode, 0) == 1:
            simt.add((mode, Hi, Wi, Ci, Co, k))
    assert simt == {(0, 4, 4, 512, 544, 3)}, simt
