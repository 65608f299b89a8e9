"""Encoder / Decoder conv stacks (reference: jukebox/vqvae/encdec.py), channels-last [N, T, C]."""
import torch.nn as nn

from .ops_cl import Conv1d, ConvTranspose1d
from .resnet import Resnet1D, use_tensor_cores


def assert_shape(x, exp_shape):
    assert tuple(x.shape) == tuple(exp_shape), f"Expected {exp_shape} got {tuple(x.shape)}"


class EncoderConvBlock(nn.Module):
    def __init__(self, input_emb_width, output_emb_width, down_t, stride_t, width, depth, m_conv,
                 dilation_growth_rate=1, dilation_cycle=None, zero_out=False, res_scale=False):
        super().__init__()
        blocks = []
        filter_t, pad_t = stride_t * 2, stride_t // 2
        if down_t > 0:
            for i in range(down_t):
                blocks.append(nn.Sequential(
                    Conv1d(input_emb_width if i == 0 else width, width, filter_t, stride_t, pad_t),
                    Resnet1D(width, depth, m_conv, dilation_growth_rate, dilation_cycle, zero_out, res_scale)))
            blocks.append(Conv1d(width, output_emb_width, 3, 1, 1))
        self.model = nn.Sequential(*blocks)

    def forward(self, x):
        for m in self.model:
            if isinstance(m, nn.Sequential):
                x = m[1](m[0](x))
            else:
                x = m(x)
        return x


class DecoderConvBock(nn.Module):
    def __init__(self, input_emb_width, output_emb_width, down_t, stride_t, width, depth, m_conv,
                 dilation_growth_rate=1, dilation_cycle=None, zero_out=False, res_scale=False,
                 reverse_decoder_dilation=False, checkpoint_res=False):
        super().__init__()
        blocks = []
        if down_t > 0:
            filter_t, pad_t = stride_t * 2, stride_t // 2
            blocks.append(Conv1d(output_emb_width, width, 3, 1, 1))
            for i in range(down_t):
                blocks.append(nn.Sequential(
                    Resnet1D(width, depth, m_conv, dilation_growth_rate, dilation_cycle, zero_out=zero_out,
                             res_scale=res_scale, reverse_dilation=reverse_decoder_dilation,
                             checkpoint_res=checkpoint_res),
                    ConvTranspose1d(width, input_emb_width if i == (down_t - 1) else width, filter_t, stride_t, pad_t)))
        self.model = nn.Sequential(*blocks)
        # decoder side: nothing downstream needs a fixed FMA order, so the residual blocks take the tensor-core kernel
        # (use_tensor_cores(module, False) gives the exact-FMA route, e.g. to compare the two)
        use_tensor_cores(self)

    def forward(self, x):
        for m in self.model:
            if isinstance(m, nn.Sequential):
                x = m[1](m[0](x))
            else:
                x = m(x)
        return x


class Encoder(nn.Module):
    def __init__(self, input_emb_width, output_emb_width, levels, downs_t, strides_t, **block_kwargs):
        super().__init__()
        self.input_emb_width, self.output_emb_width = input_emb_width, output_emb_width
        self.levels, self.downs_t, self.strides_t = levels, downs_t, strides_t
        kw = dict(block_kwargs)
        kw.pop('reverse_decoder_dilation', None)
        self.level_blocks = nn.ModuleList(
            EncoderConvBlock(input_emb_width if level == 0 else output_emb_width, output_emb_width, down_t,
                             stride_t, **kw)
            for level, down_t, stride_t in zip(range(levels), downs_t, strides_t))

    def forward(self, x):
        """x: [N, T, input_emb_width] -> list over levels of [N, T_l, output_emb_width]"""
        N, T = x.shape[0], x.shape[1]
        assert_shape(x, (N, T, self.input_emb_width))
        xs = []
        for level, down_t, stride_t in zip(range(self.levels), self.downs_t, self.strides_t):
            x = self.level_blocks[level](x)
            T = T // (stride_t ** down_t)
            assert_shape(x, (N, T, self.output_emb_width))
            xs.append(x)
        return xs


class Decoder(nn.Module):
    def __init__(self, input_emb_width, output_emb_width, levels, downs_t, strides_t, **block_kwargs):
        super().__init__()
        self.input_emb_width, self.output_emb_width = input_emb_width, output_emb_width
        self.levels, self.downs_t, self.strides_t = levels, downs_t, strides_t
        self.level_blocks = nn.ModuleList(
            DecoderConvBock(output_emb_width, output_emb_width, down_t, stride_t, **block_kwargs)
            for level, down_t, stride_t in zip(range(levels), downs_t, strides_t))
        self.out = Conv1d(output_emb_width, input_emb_width, 3, 1, 1)

    def forward(self, xs, all_levels=True):
        assert len(xs) == (self.levels if all_levels else 1)
        x = xs[-1]
        N, T = x.shape[0], x.shape[1]
        assert_shape(x, (N, T, self.output_emb_width))
        for level, down_t, stride_t in reversed(list(zip(range(self.levels), self.downs_t, self.strides_t))):
            x = self.level_blocks[level](x)
            T = T * (stride_t ** down_t)
            assert_shape(x, (N, T, self.output_emb_width))
            if level != 0 and all_levels:
                x = x + xs[level - 1]
        return self.out(x)
