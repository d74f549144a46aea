"""GPU: the condition pyramid's bilinear resize (F.interpolate, align_corners=False) in both directions -- the upsampling
kernel against torch in float64, its adjoint through the dot-product identity, and a 256^2 condition driving the 512^2
generator."""
import pytest
import torch
import torch.nn.functional as F

import golden_util as gu

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,H,W,C,s", [(2, 256, 256, 6, 2), (2, 256, 256, 6, 4), (3, 4, 8, 5, 2), (1, 1, 2, 3, 4), (2, 16, 16, 9, 8)])
def test_cond_up_matches_interpolate(cuda, B, H, W, C, s):
    from gif_b200 import ops
    x = gu.rand_uniform((B, H, W, C), B + H + C + s).to(cuda)
    y = ops.cond_up(x, s)
    ref = F.interpolate(x.double().permute(0, 3, 1, 2), size=(H * s, W * s), mode="bilinear", align_corners=False)
    assert tuple(y.shape) == (B, H * s, W * s, C)
    assert gu.rel_err(y.cpu().numpy(), ref.permute(0, 2, 3, 1).cpu().numpy()) < 1e-6


@pytest.mark.parametrize("B,H,W,C,s", [(2, 64, 64, 6, 2), (2, 64, 32, 6, 4), (3, 4, 8, 5, 2), (1, 1, 2, 3, 4)])
def test_cond_up_adjoint_identity(cuda, B, H, W, C, s):
    """<U x, y> = <x, U^T y>, and autograd runs the adjoint kernel."""
    from gif_b200 import ops
    x = gu.randn((B, H, W, C), 5).to(cuda).requires_grad_(True)
    y = gu.randn((B, H * s, W * s, C), 6).to(cuda)
    ux = ops.cond_up(x, s)
    (uty,) = torch.autograd.grad((ux * y).sum(), x)
    lhs = float((ux.double() * y.double()).sum())
    rhs = float((x.detach().double() * uty.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * max(abs(lhs), 1.0), (lhs, rhs)
    xd =x.detach().double().permute(0, 3, 1, 2).requires_grad_(True)
    (g_ref,) = torch.autograd.grad(F.interpolate(xd, size=(H * s, W * s), mode="bilinear", align_corners=False),
                                   xd, y.double().permute(0, 3, 1, 2))
    assert gu.rel_err(uty.cpu().numpy(), g_ref.permute(0, 2, 3, 1).cpu().numpy()) < 1e-6


def test_cond_resize_dispatch(cuda):
    from gif_b200 import ops
    x = gu.rand_uniform((2, 64, 64, 6), 7).to(cuda)
    assert ops.cond_resize(x, 64) is x
    assert torch.equal(ops.cond_resize(x, 16), ops.cond_down(x, 4))
    assert torch.equal(ops.cond_resize(x, 256), ops.cond_up(x, 4))
    with pytest.raises(NotImplementedError):
        ops.cond_resize(x, 48)
    with pytest.raises(NotImplementedError):
        ops.cond_resize(gu.rand_uniform((2, 96, 96, 6), 8).to(cuda), 32)


def test_generator_512_with_256_condition(cuda, tf32_mode):
    """step 7 (512^2) fed a 256^2 condition, as the texture-interpolation loss does at 512^2: no longer raises."""
    from gif_b200.model.stg2_generator import StyledGenerator
    G = StyledGenerator(embedding_vocab_size=16, rendered_flame_ascondition=True, normal_maps_as_cond=True).to(cuda)
    with torch.no_grad():
        img = G(gu.rand_uniform((2, 6, 256, 256), 9).to(cuda), step=7, input_indices=gu.randint(16, (2,), 10).to(cuda))[0]
    assert tuple(img.shape) == (2, 3, 512, 512) and bool(torch.isfinite(img).all())
    with pytest.raises(NotImplementedError):
        G(gu.rand_uniform((2, 6, 96, 96), 9).to(cuda), step=7, input_indices=gu.randint(16, (2,), 10).to(cuda))
