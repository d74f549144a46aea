"""Operator library with the API of the reference's model/stylegan2_common_layers.py ("cl.py").

Every class keeps the reference's name, constructor signature, parameter/buffer names and shapes (so reference
checkpoints load, SURVEY 8b) and its NCHW tensor interface; the arithmetic runs on the sm_100a kernels of
libgifb200.so through gif_b200.ops (channels-last internally; the NCHW tensors these modules return are views of
channels-last storage, so chaining modules costs no layout conversions).

Formulation of ModulatedConv2d (cl.py:250-349): instead of materialising a per-sample weight (B,Co,Ci,k,k) and
running a grouped convolution, the style modulates the *input* (x * s[b,i]), one shared-weight convolution runs on
the tensor cores, and the demodulation coefficient d[b,o] scales the *output* (SURVEY Appendix A3; equal to the
reference to fp32 rounding).
"""
import math
import random

import torch
from torch import nn
from torch.nn import functional as F

from .. import ops


# --------------------------------------------------------------------------------------------- helpers
def make_kernel(k):
    """cl.py:83-91."""
    k = torch.tensor(k, dtype=torch.float32)
    if k.ndim == 1:
        k = k[None, :] * k[:, None]
    k /= k.sum()
    return k


def upfirdn2d(input, kernel, up=1, down=1, pad=(0, 0)):
    """cl.py:42-72 (NCHW in, NCHW view out)."""
    return ops.to_nchw_view(ops.upfirdn2d(ops.to_nhwc(input), kernel, up=up, down=down, pad=pad))


class FusedLeakyReLU(nn.Module):
    """cl.py:22-39: scale * leaky_relu(x + bias)."""

    def __init__(self, channel, negative_slope=0.2, scale=2 ** 0.5):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(1, channel, 1, 1))
        self.negative_slope = negative_slope
        self.scale = scale

    def forward(self, input, _rt=False):
        return ops.to_nchw_view(ops.bias_act(ops.to_nhwc(input), self.bias, self.negative_slope, self.scale, rt=_rt))


class PixelNorm(nn.Module):
    """cl.py:75-80 (a (B,512) vector op: plain torch glue)."""

    def forward(self, input):
        return input * torch.rsqrt(torch.mean(input ** 2, dim=1, keepdim=True) + 1e-8)


class Upsample(nn.Module):
    """cl.py:94-112."""

    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        kernel = make_kernel(kernel) * (factor ** 2)
        self.register_buffer('kernel', kernel)
        p = kernel.shape[0] - factor
        self.pad = ((p + 1) // 2 + factor - 1, p // 2)

    def forward(self, input):
        return upfirdn2d(input, self.kernel, up=self.factor, down=1, pad=self.pad)


class Downsample(nn.Module):
    """cl.py:115-133."""

    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        kernel = make_kernel(kernel)
        self.register_buffer('kernel', kernel)
        p = kernel.shape[0] - factor
        self.pad = ((p + 1) // 2, p // 2)

    def forward(self, input):
        return upfirdn2d(input, self.kernel, up=1, down=self.factor, pad=self.pad)


class Blur(nn.Module):
    """cl.py:136-152."""

    def __init__(self, kernel, pad, upsample_factor=1):
        super().__init__()
        kernel = make_kernel(kernel)
        if upsample_factor > 1:
            kernel = kernel * (upsample_factor ** 2)
        self.register_buffer('kernel', kernel)
        self.pad = pad

    def forward(self, input):
        return upfirdn2d(input, self.kernel, pad=self.pad)


def _conv_mode(kernel_size, stride, padding):
    if stride == 1 and padding == kernel_size // 2:
        return ops.S1
    if stride == 2 and padding == 0:
        return ops.S2
    raise NotImplementedError(f"gif_b200 convolution: (k={kernel_size}, stride={stride}, padding={padding}) is not on "
                              "the GIF hot path (supported: stride 1 with 'same' padding, stride 2 without padding)")


def _pad_channels_for_tc(x, wt):
    """tensor-core modes (tf32 / bf16x3): zero-pad the input channels (and the weight's Ci) to a multiple of 32 so that odd-channel layers (the
    9-channel discriminator stem, the 513-channel minibatch-stddev conv) run on the tensor-core kernels; values unchanged."""
    ci = x.shape[-1]
    if ops.tc_enabled() and ci % 32 != 0 and wt.shape[1] % 32 == 0:
        pad = 32 - ci % 32
        x = F.pad(x, (0, pad))
        wt = F.pad(wt, (0, pad))
    return x, wt


class EqualConv2d(nn.Module):
    """cl.py:155-190."""

    def __init__(self, in_channel, out_channel, kernel_size, stride=1, padding=0, bias=True):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_channel, in_channel, kernel_size, kernel_size))
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.stride = stride
        self.padding = padding
        self.kernel_size = kernel_size
        self.bias = nn.Parameter(torch.zeros(out_channel)) if bias else None

    def forward_nhwc(self, x):
        mode = _conv_mode(self.kernel_size, self.stride, self.padding)
        wt = ops.prep_weight(self.weight, self.scale)
        x, wt = _pad_channels_for_tc(x, wt)
        if self.bias is not None:
            return ops.conv2d_bias_act(x, wt, self.bias, self.kernel_size, mode, slope=1.0, gain=1.0)
        return ops.conv2d(x, wt, self.kernel_size, mode)

    def forward(self, input):
        return ops.to_nchw_view(self.forward_nhwc(ops.to_nhwc(input)))

    def __repr__(self):
        return (f'{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]},'
                f' {self.weight.shape[2]}, stride={self.stride}, padding={self.padding})')


class EqualLinear(nn.Module):
    """cl.py:193-235."""

    def __init__(self, in_dim, out_dim, bias=True, bias_init=0, lr_mul=1, activation=None, scale_weight=1.0,
                 apply_sqrt2_fac_in_eq_lin=False):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_dim, in_dim).div_(lr_mul / scale_weight))
        self.bias = nn.Parameter(torch.zeros(out_dim).fill_(bias_init)) if bias else None
        self.activation = activation
        self.scale = (1 / math.sqrt(in_dim)) * lr_mul
        self.lr_mul = lr_mul
        self.apply_sqrt2_fac_in_eq_lin = apply_sqrt2_fac_in_eq_lin

    def forward(self, input):
        x = input.reshape(-1, input.shape[-1])
        y = ops.matmul(x, self.weight, trans_b=True, alpha=self.scale)
        bias = None if self.bias is None else self.bias * self.lr_mul
        if self.activation:
            gain = 1.41421356237 if self.apply_sqrt2_fac_in_eq_lin else 1.0      # cl.py:221-222
            y = ops.bias_act(y, bias, slope=0.2, gain=gain)
        elif bias is not None:
            y = ops.bias_act(y, bias, slope=1.0, gain=1.0)
        return y.reshape(input.shape[:-1] + (self.weight.shape[0],))

    def __repr__(self):
        return f'{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]})'


class ScaledLeakyReLU(nn.Module):
    """cl.py:238-247."""

    def __init__(self, negative_slope=0.2):
        super().__init__()
        self.negative_slope = negative_slope

    def forward(self, input):
        return ops.to_nchw_view(ops.bias_act(ops.to_nhwc(input), None, self.negative_slope, math.sqrt(2)))


class ModulatedConv2d(nn.Module):
    """cl.py:250-349."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, demodulate=True, upsample=False,
                 downsample=False, blur_kernel=[1, 3, 3, 1], apply_sqrt2_fac_in_eq_lin=False):
        super().__init__()
        self.eps = 1e-8
        self.kernel_size = kernel_size
        self.in_channel = in_channel
        self.out_channel = out_channel
        self.upsample = upsample
        self.downsample = downsample
        if upsample:
            factor = 2
            p = (len(blur_kernel) - factor) - (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2 + factor - 1, p // 2 + 1), upsample_factor=factor)
        if downsample:
            factor = 2
            p = (len(blur_kernel) - factor) + (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2, p // 2))
        fan_in = in_channel * kernel_size ** 2
        self.scale = 1 / math.sqrt(fan_in)
        self.padding = kernel_size // 2
        self.weight = nn.Parameter(torch.randn(1, out_channel, in_channel, kernel_size, kernel_size))
        self.modulation = EqualLinear(style_dim, in_channel, bias_init=1,
                                      apply_sqrt2_fac_in_eq_lin=apply_sqrt2_fac_in_eq_lin)
        self.demodulate = demodulate

    def __repr__(self):
        return (f'{self.__class__.__name__}({self.in_channel}, {self.out_channel}, {self.kernel_size}, '
                f'upsample={self.upsample}, downsample={self.downsample})')

    def accumulate(self, x, style):
        """NHWC x -> (acc, d): the un-demodulated shared-weight convolution of the modulated input (after the blur
        of the upsample branch) and the demodulation coefficients d[b,o] (None if demodulate=False)."""
        s = self.modulation(style)                                        # (B,Ci)  cl.py:311
        wt = ops.prep_weight(self.weight[0], self.scale)                  # (T,Co,Ci) = W~ tap-major
        k = self.kernel_size
        if k == 1 and self.out_channel == 3 and not (self.upsample or self.downsample):
            # ToRGB: per-sample 1x1 weights ws[b,c,i] = W~[c,i] s[b,i] (3*Ci numbers per sample), no modulated copy of x
            acc = ops.torgb(x, wt[0][None] * s[:, None, :])
        else:
            if self.upsample:
                acc = ops.modconv(x, s, wt, k, ops.T2)                    # (2H+1)^2  cl.py:322-331
                acc = ops.upfirdn2d(acc, self.blur.kernel, pad=self.blur.pad)   # cl.py:333
            elif self.downsample:
                xs = ops.chan_scale(x, s, ops.tf32_enabled())
                xs = ops.upfirdn2d(xs, self.blur.kernel, pad=self.blur.pad, rt=ops.tf32_enabled())
                acc = ops.conv2d(xs, wt, k, ops.S2)                       # cl.py:335-341
            else:
                acc = ops.modconv(x, s, wt, k, ops.S1)                    # cl.py:343-347
        d = None
        if self.demodulate:
            q = (wt * wt).sum(dim=0)                                      # (Co,Ci) = sum_taps W~^2
            d = ops.demod(s, q, self.eps)                                 # cl.py:315-316
        return acc, d

    def forward_nhwc(self, x, style):
        acc, d = self.accumulate(x, style)
        return acc if d is None else ops.chan_scale(acc, d)

    def forward(self, input, style):
        return ops.to_nchw_view(self.forward_nhwc(ops.to_nhwc(input), style))


class NoiseInjection(nn.Module):
    """cl.py:388-431: image + Conv3x3(ReLU(Conv3x3(ReLU(Conv3x3(cond))))) with plain nn.Conv2d parameters."""

    @staticmethod
    def small_init_weights(m):
        if hasattr(m, 'weight'):
            m.weight.data = torch.randn_like(m.weight) / 100
        if hasattr(m, 'bias'):
            m.bias.data.fill_(0.0001)

    def __init__(self, noise_in_chalnnels, noise_out_channels):
        super().__init__()
        self.noise_in_chalnnels = noise_in_chalnnels
        c = noise_in_chalnnels
        self.noise_conv = nn.Sequential(
            nn.Conv2d(in_channels=c, out_channels=2 * c, kernel_size=3, padding=1, dilation=1),
            nn.ReLU(),
            nn.Conv2d(in_channels=2 * c, out_channels=4 * c, kernel_size=3, padding=1, dilation=1),
            nn.ReLU(),
            nn.Conv2d(in_channels=4 * c, out_channels=noise_out_channels, kernel_size=3, padding=1, dilation=1),
        )
        self.noise_conv.apply(NoiseInjection.small_init_weights)

    def convolved_noise_nhwc(self, noise):
        """noise (B,r,r,c) NHWC -> (B,r,r,Co) NHWC *without* the last bias (returned separately for fusion).

        In tf32 mode the 6/12/24-channel tensors are zero-padded to 32 channels (weights and biases padded to match, so
        the values are unchanged) which makes all three convolutions eligible for the tensor-core kernel: 5x more nominal
        FLOPs on the first one, but on a pipe that is ~50x faster than the fp32 SIMT path."""
        c0, c2, c4 = self.noise_conv[0], self.noise_conv[2], self.noise_conv[4]
        w0, w2, w4 = ops.prep_weight(c0.weight), ops.prep_weight(c2.weight), ops.prep_weight(c4.weight)
        b0, b2 = c0.bias, c2.bias
        if ops.tc_enabled() and noise.shape[1] >= 4 and (noise.shape[1] & (noise.shape[1] - 1)) == 0:
            def up32(n):
                return (n + 31) // 32 * 32
            ci, c1, c2n = w0.shape[2], w0.shape[1], w2.shape[1]
            noise = F.pad(noise, (0, up32(ci) - ci))
            w0 = F.pad(w0, (0, up32(ci) - ci, 0, up32(c1) - c1))
            b0 = F.pad(b0, (0, up32(c1) - c1))
            w2 = F.pad(w2, (0, up32(c1) - c1, 0, up32(c2n) - c2n))
            b2 = F.pad(b2, (0, up32(c2n) - c2n))
            w4 = F.pad(w4, (0, up32(c2n) - c2n))
        rt = ops.tf32_enabled()
        h = ops.conv2d_bias_act(noise, w0, b0, 3, ops.S1, slope=0.0, gain=1.0, rt=rt)   # conv + bias + ReLU, one kernel
        h = ops.conv2d_bias_act(h, w2, b2, 3, ops.S1, slope=0.0, gain=1.0, rt=rt)
        h = ops.conv2d(h, w4, 3, ops.S1)
        return h, c4.bias

    def forward(self, image, noise):
        x = ops.to_nhwc(image)
        if noise is None:
            b, _, hh, ww = image.shape
            noise = image.new_empty(b, self.noise_in_chalnnels, hh, ww).normal_()
        h, b4 = self.convolved_noise_nhwc(ops.to_nhwc(noise))
        # image + (h + bias): one fused pass (identity activation)
        return ops.to_nchw_view(ops.bias_act(h, b4, slope=1.0, gain=1.0, add=x))


class ConstantInput(nn.Module):
    """cl.py:434-444."""

    def __init__(self, channel, size=4):
        super().__init__()
        self.input = nn.Parameter(torch.randn(1, channel, size, size))

    def forward(self, input):
        return self.input.repeat(input.shape[0], 1, 1, 1)


class StyledConv(nn.Module):
    """cl.py:447-486: ModulatedConv2d -> NoiseInjection(cond) -> FusedLeakyReLU; the demodulation, the noise add, the
    bias and the activation are ONE kernel (gifb200_bias_act) on the convolution's accumulator."""

    def __init__(self, in_channel, out_channel, kernel_size, noise_in_dims, style_dim=512, upsample=False,
                 blur_kernel=[1, 3, 3, 1], demodulate=True, apply_sqrt2_fac_in_eq_lin=False):
        super().__init__()
        self.conv = ModulatedConv2d(in_channel, out_channel, kernel_size, style_dim, upsample=upsample,
                                    blur_kernel=blur_kernel, demodulate=demodulate,
                                    apply_sqrt2_fac_in_eq_lin=apply_sqrt2_fac_in_eq_lin)
        self.noise = NoiseInjection(noise_in_dims, out_channel)
        self.activate = FusedLeakyReLU(out_channel)

    def forward_nhwc(self, x, style, noise_nhwc):
        acc, d = self.conv.accumulate(x, style)
        if noise_nhwc is None:
            b, hh, ww, _ = acc.shape
            noise_nhwc = acc.new_empty(b, hh, ww, self.noise.noise_in_chalnnels).normal_()
        h, b4 = self.noise.convolved_noise_nhwc(noise_nhwc)
        bias = self.activate.bias.reshape(-1) + b4                        # last noise-conv bias folds into the act bias
        return ops.bias_act(acc, bias, self.activate.negative_slope, self.activate.scale, rowscale=d, add=h)

    def forward(self, input, style, noise=None):
        n = None if noise is None else ops.to_nhwc(noise)
        return ops.to_nchw_view(self.forward_nhwc(ops.to_nhwc(input), style, n))


class ToRGB(nn.Module):
    """cl.py:489-511."""

    def __init__(self, in_channel, style_dim, upsample=True, blur_kernel=[1, 3, 3, 1],
                 apply_sqrt2_fac_in_eq_lin=False):
        super().__init__()
        if upsample:
            self.upsample = Upsample(blur_kernel)
        self.conv = ModulatedConv2d(in_channel, 3, 1, style_dim, demodulate=False,
                                    apply_sqrt2_fac_in_eq_lin=apply_sqrt2_fac_in_eq_lin)
        self.bias = nn.Parameter(torch.zeros(1, 3, 1, 1))

    def forward_nhwc(self, x, style, skip):
        acc, _ = self.conv.accumulate(x, style)
        if skip is not None:
            skip = ops.upfirdn2d(skip, self.upsample.kernel, up=self.upsample.factor, pad=self.upsample.pad)
        return ops.bias_act(acc, self.bias, slope=1.0, gain=1.0, add=skip)   # + bias (+ upsampled skip), one pass

    def forward(self, input, style, skip=None):
        s = None if skip is None else ops.to_nhwc(skip)
        return ops.to_nchw_view(self.forward_nhwc(ops.to_nhwc(input), style, s))


def get_w_frm_z(n_mlp, style_dim, lr_mlp=1, scale_weight=1.0):
    """cl.py:514-533."""
    if n_mlp > 0:
        layers = [PixelNorm()]
        for _ in range(n_mlp):
            layers.append(EqualLinear(style_dim, style_dim, lr_mul=lr_mlp, activation='fused_lrelu',
                                      scale_weight=scale_weight))
        return nn.Sequential(*layers)

    class Net(nn.Module):
        def forward(self, *args):
            return args[0]

    return Net()


class Generator(nn.Module):
    """cl.py:536-750: the plain StyleGAN2 synthesis stack (constant input, StyledConv pairs with single-channel noise inputs,
    ToRGB skips).  Not used by GIF's training path (train.py builds ``model.stg2_generator.StyledGenerator``), and the
    reference's own constructor cannot run (cl.py:569-571 passes ``style_dim`` positionally into StyledConv's
    ``noise_in_dims`` slot AND ``noise_in_dims=1`` by keyword: TypeError), so its outputs are unpinned; this follows the
    evident intent so that everything the reference's operator module exports is importable and runnable from this one.  Same attribute / state_dict
    names (``style``, ``input``, ``conv1``, ``to_rgb1``, ``convs``, ``to_rgbs``, ``noises.noise_{i}``)."""

    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=[1, 3, 3, 1], lr_mlp=0.01):
        super().__init__()
        self.size = size
        self.style_dim = style_dim
        self.style = get_w_frm_z(n_mlp, style_dim, lr_mlp)
        m = channel_multiplier
        self.channels = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * m, 128: 128 * m, 256: 64 * m, 512: 32 * m, 1024: 16 * m}
        self.log_size = int(math.log(size, 2))
        self.num_layers = (self.log_size - 2) * 2 + 1
        self.n_latent = self.log_size * 2 - 2
        width = self.channels[4]
        self.input = ConstantInput(width)
        self.conv1 = StyledConv(width, width, 3, style_dim=style_dim, blur_kernel=blur_kernel, noise_in_dims=1)
        self.to_rgb1 = ToRGB(width, style_dim, upsample=False)
        self.convs, self.upsamples, self.to_rgbs, self.noises = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.Module()
        for layer in range(self.num_layers):
            r = 2 ** ((layer + 5) // 2)
            self.noises.register_buffer(f'noise_{layer}', torch.randn(1, 1, r, r))
        for octave in range(3, self.log_size + 1):
            nxt = self.channels[2 ** octave]
            self.convs.append(StyledConv(width, nxt, 3, style_dim=style_dim, upsample=True, blur_kernel=blur_kernel,
                                         noise_in_dims=1))
            self.convs.append(StyledConv(nxt, nxt, 3, style_dim=style_dim, blur_kernel=blur_kernel, noise_in_dims=1))
            self.to_rgbs.append(ToRGB(nxt, style_dim))
            width = nxt

    def make_noise(self):
        dev = self.input.input.device
        sizes = [4] + [2 ** o for o in range(3, self.log_size + 1) for _ in range(2)]
        return [torch.randn(1, 1, r, r, device=dev) for r in sizes]

    def mean_latent(self, n_latent):
        return self.style(torch.randn(n_latent, self.style_dim, device=self.input.input.device)).mean(0, keepdim=True)

    def get_latent(self, input):
        return self.style(input)

    def _latents(self, styles, inject_index):
        """cl.py:690-708: one w per layer; two styles are crossed over at ``inject_index``."""
        if len(styles) < 2:
            return styles[0].unsqueeze(1).repeat(1, self.n_latent, 1) if styles[0].ndim < 3 else styles[0]
        if inject_index is None:
            inject_index = random.randint(1, self.n_latent - 1)
        return torch.cat([styles[0].unsqueeze(1).repeat(1, inject_index, 1),
                          styles[1].unsqueeze(1).repeat(1, self.n_latent - inject_index, 1)], 1)

    def forward(self, styles, return_latents=False, inject_index=None, truncation=1, truncation_latent=None,
                input_is_latent=False, noise=None, randomize_noise=True):
        if not input_is_latent:
            styles = [self.style(s) for s in styles]
        if noise is None:
            noise = [None] * self.num_layers if randomize_noise else \
                [getattr(self.noises, f'noise_{i}') for i in range(self.num_layers)]
        if truncation < 1:
            styles = [truncation_latent + truncation * (s - truncation_latent) for s in styles]
        latent = self._latents(styles, inject_index)
        batch = latent.shape[0]

        def per_sample(n):          # stored noises are (1,1,r,r): one map shared by the batch
            return None if n is None else ops.to_nhwc(n.expand(batch, -1, -1, -1))
        x = ops.to_nhwc(self.input(latent))
        x = self.conv1.forward_nhwc(x, latent[:, 0], per_sample(noise[0]))
        skip = self.to_rgb1.forward_nhwc(x, latent[:, 1], None)
        for j, to_rgb in enumerate(self.to_rgbs):
            i = 1 + 2 * j
            x = self.convs[2 * j].forward_nhwc(x, latent[:, i], per_sample(noise[i]))
            x = self.convs[2 * j + 1].forward_nhwc(x, latent[:, i + 1], per_sample(noise[i + 1]))
            skip = to_rgb.forward_nhwc(x, latent[:, i + 2], skip)
        image = ops.to_nchw_view(skip)
        return (image, latent) if return_latents else (image, None)


class ConvLayer(nn.Sequential):
    """cl.py:752-799: [Blur ->] EqualConv2d -> FusedLeakyReLU | ScaledLeakyReLU."""

    def __init__(self, in_channel, out_channel, kernel_size, downsample=False, blur_kernel=[1, 3, 3, 1], bias=True,
                 activate=True):
        layers = []
        if downsample:
            factor = 2
            p = (len(blur_kernel) - factor) + (kernel_size - 1)
            layers.append(Blur(blur_kernel, pad=((p + 1) // 2, p // 2)))
            stride = 2
            self.padding = 0
        else:
            stride = 1
            self.padding = kernel_size // 2
        layers.append(EqualConv2d(in_channel, out_channel, kernel_size, padding=self.padding, stride=stride,
                                  bias=bias and not activate))
        if activate:
            layers.append(FusedLeakyReLU(out_channel) if bias else ScaledLeakyReLU(0.2))
        super().__init__(*layers)

    def forward_nhwc(self, x, rt_out=False):
        """Channels-last fast path used by ResBlock / Discriminator (same arithmetic as the Sequential): the blur is one
        upfirdn2d pass, and convolution + bias + leaky-ReLU*sqrt(2) is ONE kernel (fused epilogue)."""
        tf32 = ops.tf32_enabled()
        layers = list(self)
        i = 0
        if isinstance(layers[0], Blur):
            blur, conv = layers[0], layers[1]
            if conv.kernel_size == 1:
                # blur(pad 1,1) then 1x1 stride-2 conv == FIR evaluated only at the even output sites
                # (upfirdn2d down=2), then a stride-1 1x1 conv: 4x fewer FIR outputs (cl.py:765-771,:776-786)
                x = ops.upfirdn2d(x, blur.kernel, down=2, pad=blur.pad, rt=tf32)
            else:
                x = ops.upfirdn2d(x, blur.kernel, pad=blur.pad, rt=tf32)
            i = 1
        conv = layers[i]
        act = layers[i + 1] if i + 1 < len(layers) else None
        k = conv.kernel_size
        mode = ops.S1 if (k == 1 and conv.stride == 2) else _conv_mode(k, conv.stride, conv.padding)
        xp, wt = _pad_channels_for_tc(x, ops.prep_weight(conv.weight, conv.scale))
        if isinstance(act, FusedLeakyReLU):
            return ops.conv2d_bias_act(xp, wt, act.bias, k, mode, act.negative_slope, act.scale, rt=rt_out and tf32)
        if isinstance(act, ScaledLeakyReLU):
            return ops.conv2d_bias_act(xp, wt, None, k, mode, act.negative_slope, math.sqrt(2), rt=rt_out and tf32)
        if conv.bias is not None:
            return ops.conv2d_bias_act(xp, wt, conv.bias, k, mode, slope=1.0, gain=1.0)
        return ops.conv2d(xp, wt, k, mode)

    def forward(self, input):
        return ops.to_nchw_view(self.forward_nhwc(ops.to_nhwc(input)))


class ResBlock(nn.Module):
    """cl.py:802-820."""

    def __init__(self, in_channel, out_channel, blur_kernel=[1, 3, 3, 1]):
        super().__init__()
        self.conv1 = ConvLayer(in_channel, in_channel, 3)
        self.conv2 = ConvLayer(in_channel, out_channel, 3, downsample=True)
        self.skip = ConvLayer(in_channel, out_channel, 1, downsample=True, activate=False, bias=False)

    def forward_nhwc(self, x):
        out = self.conv2.forward_nhwc(self.conv1.forward_nhwc(x))
        skip = self.skip.forward_nhwc(x)
        return ops.axpby(out, skip, 1 / math.sqrt(2), 1 / math.sqrt(2), rt=ops.tf32_enabled())

    def forward(self, input):
        return ops.to_nchw_view(self.forward_nhwc(ops.to_nhwc(input)))
