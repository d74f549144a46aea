"""GIF generator with the API of the reference's model/stg2_generator.py ("gen.py"): identity embedding -> 8-layer
z->w mapping -> StyleGAN2 synthesis blocks at 4..256 (1024) with the 6-channel FLAME render injected as the
"noise" input of every StyledConv.  Same class names, constructor / forward signatures and state_dict keys.

``FlameTextureSpace`` (gen.py:336-421, imported from here by loss_functions/losses.py:9) is re-exported from
``gif_b200.texture_space`` at the bottom of this file.
"""
import random

import numpy as np
import torch
from torch import nn

from .. import ops
from .stylegan2_common_layers import StyledConv, ToRGB, get_w_frm_z


class ConstantInput(nn.Module):
    """gen.py:21-31."""

    def __init__(self, channel, size=4, constant_background=False):
        super().__init__()
        self.input = nn.Parameter(torch.randn(1, channel, size, size))

    def forward(self, input):
        return self.input.repeat(input.shape[0], 1, 1, 1)


class ImgEmbedding(nn.Module):
    """gen.py:34-46: a frozen (buffer) identity embedding."""

    def __init__(self, vector_size, vocab_size=70_000):
        super().__init__()
        self.register_buffer('embd_weight', torch.randn((vocab_size, vector_size)))

    def get_embddings(self):
        return self.embd_weight

    def forward(self, input):
        return self.embd_weight[input]


class StyledConvStyleGAN2(nn.Module):
    """gen.py:48-66."""

    def __init__(self, in_chnl, out_chnl, ker_sz, blur_kernel, noise_in_dims, one_conv_block=False,
                 apply_sqrt2_fac_in_eq_lin=False):
        super().__init__()
        self.one_conv_block = one_conv_block
        self.st_cv1 = StyledConv(in_chnl, out_chnl, ker_sz, upsample=not self.one_conv_block, blur_kernel=blur_kernel,
                                 noise_in_dims=noise_in_dims, apply_sqrt2_fac_in_eq_lin=apply_sqrt2_fac_in_eq_lin)
        if not self.one_conv_block:
            self.st_cv2 = StyledConv(out_chnl, out_chnl, ker_sz, upsample=False, blur_kernel=blur_kernel,
                                     noise_in_dims=noise_in_dims, apply_sqrt2_fac_in_eq_lin=apply_sqrt2_fac_in_eq_lin)

    def forward_nhwc(self, x, style, noise_nhwc):
        x = self.st_cv1.forward_nhwc(x, style, noise_nhwc)
        if self.one_conv_block:
            return x
        return self.st_cv2.forward_nhwc(x, style, noise_nhwc)

    def forward(self, input, style, noise=None):
        n = None if noise is None else ops.to_nhwc(noise)
        return ops.to_nchw_view(self.forward_nhwc(ops.to_nhwc(input), style, n))


class Generator(nn.Module):
    """gen.py:69-209."""

    def __init__(self, code_dim, core_tensor_res=4, channel_multiplier=2, noise_in_dims=None,
                 apply_sqrt2_fac_in_eq_lin=False):
        super().__init__()
        assert core_tensor_res < 64
        assert code_dim == 512
        m = channel_multiplier
        self.start_step = int(np.log2(core_tensor_res)) - 2
        self.const_input = ConstantInput(512, size=core_tensor_res)
        blur_kernel = [1, 3, 3, 1]
        chans = [512, 512, 512, 512, 256 * m, 128 * m, 64 * m, 32 * m, 16 * m]          # gen.py:84-113
        kw = dict(blur_kernel=blur_kernel, noise_in_dims=noise_in_dims,
                  apply_sqrt2_fac_in_eq_lin=apply_sqrt2_fac_in_eq_lin)
        blocks = [StyledConvStyleGAN2(code_dim, chans[0], 3, one_conv_block=True, **kw)]
        for i in range(1, 9):
            blocks.append(StyledConvStyleGAN2(chans[i - 1], chans[i], 3, **kw))
        self.progression = nn.ModuleList(blocks)
        self.to_rgb = nn.ModuleList(
            [ToRGB(chans[i], code_dim, upsample=i > 0, apply_sqrt2_fac_in_eq_lin=apply_sqrt2_fac_in_eq_lin)
             for i in range(9)])

    def forward(self, style, pose, noise, step=0, alpha=-1, input_indices=None, mixing_range=(-1, -1)):
        out = torch.zeros((noise[0].shape[0], 3), device=noise[0].device) if pose is None else pose
        if len(style) < 2:
            inject_index = [len(self.progression) + 1]
        else:
            inject_index = random.sample(list(range(step)), len(style) - 1)
        crossover = 0
        rgb = None
        x = None
        for i in range(self.start_step, len(self.progression)):
            if mixing_range == (-1, -1):
                if crossover < len(inject_index) and i > inject_index[crossover]:
                    crossover = min(crossover + 1, len(style))
                style_step = style[crossover]
            else:
                style_step = style[1] if mixing_range[0] <= i <= mixing_range[1] else style[0]
            if i == self.start_step:
                x = ops.to_nhwc(self.const_input(out))
            x = self.progression[i].forward_nhwc(x, style_step, ops.to_nhwc(noise[i]))
            rgb = self.to_rgb[i].forward_nhwc(x, style_step, rgb)
            if i == step:
                break
        return [ops.to_nchw_view(rgb)]     # a one-element list, as the reference returns (gen.py:209)


class StyledGenerator(nn.Module):
    """gen.py:212-333."""

    def __init__(self, n_mlp=8, embedding_vocab_size=1, rendered_flame_ascondition=False, normal_maps_as_cond=False,
                 core_tensor_res=4, w_truncation_factor=1.0, apply_sqrt2_fac_in_eq_lin=False):
        super().__init__()
        noise_in_dims = int(rendered_flame_ascondition * 3 + normal_maps_as_cond * 3)
        self.core_tensor_res = core_tensor_res
        self.rendered_flame_ascondition = rendered_flame_ascondition
        self.normal_maps_as_cond = normal_maps_as_cond
        self.w_truncation_factor = w_truncation_factor
        self.mean_w = None
        code_dim = 512
        self.generator = Generator(code_dim, core_tensor_res=core_tensor_res, noise_in_dims=noise_in_dims,
                                   apply_sqrt2_fac_in_eq_lin=apply_sqrt2_fac_in_eq_lin)
        self.embedding_vocab_size = embedding_vocab_size
        if embedding_vocab_size > 1:
            self.image_embedding = ImgEmbedding(vector_size=code_dim, vocab_size=self.embedding_vocab_size)
            self.img_embdng = self.image_embedding      # the reference registers the same module twice (gen.py:229-231)
        self.z_to_w = get_w_frm_z(n_mlp, style_dim=code_dim, lr_mlp=0.01, scale_weight=1.0)

    def get_embddings(self):
        return self.image_embedding.get_embddings()

    def forward(self, input, pose=None, noise=None, step=9, alpha=1, mean_style=None, style_weight=0,
                input_indices=None, mixing_range=(-1, -1)):
        assert step > np.log2(self.core_tensor_res) - 2
        styles = []
        if type(input) not in (list, tuple):
            input = [input]
        if self.rendered_flame_ascondition or self.normal_maps_as_cond:
            if input_indices is None:
                input_indices = torch.zeros(input[0].shape[0], dtype=torch.long, device=input[0].device)
            if input_indices.dtype == torch.float32:                     # the caller feeds z directly (gen.py:272)
                styles.append(self.z_to_w(input_indices))
            else:
                w = self.z_to_w(self.img_embdng(input_indices))
                if np.abs(self.w_truncation_factor - 1.0) > 0.01:
                    if self.mean_w is None:
                        self.mean_w = torch.mean(self.z_to_w(self.get_embddings()), dim=0)
                    styles.append(w + (self.mean_w - w) * (1.0 - self.w_truncation_factor))
                else:
                    styles.append(w)
        else:
            for inp in input:
                if self.embedding_vocab_size > 1:
                    if input_indices.dtype == torch.float32:
                        styles.append(torch.cat([inp, input_indices], dim=1))
                    else:
                        styles.append(torch.cat([inp, self.img_embdng(input_indices)], dim=1))
                else:
                    styles.append(inp)
        batch = input[0].shape[0]
        if noise is None:
            noise = [torch.zeros(batch, 3, 4 * 2 ** i, 4 * 2 ** i, device=input[0].device) for i in range(step + 1)]
        if self.rendered_flame_ascondition or self.normal_maps_as_cond:
            # condition pyramid (gen.py:309-314): bilinear, align_corners=False, power-of-two reductions and enlargements
            cond = ops.to_nhwc(input[0])
            noise = list(noise)
            for i in range(step + 1):
                noise[i] = ops.to_nchw_view(ops.cond_resize(cond, 4 * 2 ** i))
        if mean_style is not None:
            styles = [mean_style + style_weight * (style - mean_style) for style in styles]
        return self.generator(styles, pose, noise, step, alpha, input_indices=input_indices, mixing_range=mixing_range)


# loss_functions/losses.py:9 does ``from model.stg2_generator import FlameTextureSpace`` (class at gen.py:336); the
# implementation (fused texture-stealing kernel + adjoint) lives in gif_b200/texture_space.py.
from ..texture_space import FlameTextureSpace  # noqa: E402,F401
