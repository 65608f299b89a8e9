"""Dilated residual stacks (reference: jukebox/vqvae/resnet.py:27-75), channels-last."""
import math

import torch as t
import torch.nn as nn

from .._lib import lib, check, ptr, stream_ptr
from .ops_cl import Conv1d, ReLU


class ResConv1DBlock(nn.Module):
    """x + res_scale * Conv1x1(ReLU(Conv3_dilated(ReLU(x)))) - one fused launch for C in (32, 64) with
    n_state == n_in, otherwise two fused-epilogue conv launches."""

    def __init__(self, n_in, n_state, dilation=1, zero_out=False, res_scale=1.0):
        super().__init__()
        self.model = nn.Sequential(ReLU(), Conv1d(n_in, n_state, 3, 1, dilation, dilation),
                                   ReLU(), Conv1d(n_state, n_in, 1, 1, 0))
        if zero_out:
            nn.init.zeros_(self.model[-1].weight)
            nn.init.zeros_(self.model[-1].bias)
        self.res_scale = res_scale
        # decoder-side stacks (Decoder, Conditioner) run this block on the tensor cores (fp16 x 3 split, jk_resblock_tc);
        # the encoder feeds the bit-exact codebook argmin and keeps the exact-FMA kernel.  Set by `use_tensor_cores`.
        self.tensor_cores = False

    def forward(self, x):
        c3, c1 = self.model[1], self.model[3]
        if c3.n_in == c3.n_out and c3.n_in in (32, 64):
            # the VQ-VAE's own shapes: ONE launch, the hidden activation stays in shared memory
            x = x.contiguous()
            n, T, C_ = x.shape
            (w1, b1), (w2, b2) = c3.packed(), c1.packed()
            out = t.empty_like(x)
            if self.tensor_cores:
                check(lib().jk_resblock_tc(ptr(x), ptr(out), ptr(w1), ptr(b1), ptr(w2), ptr(b2), n, T, C_, c3.dilation,
                                           float(self.res_scale), stream_ptr()))
            else:
                check(lib().jk_resblock_cl(ptr(x), ptr(out), None, ptr(w1), ptr(b1), ptr(w2), ptr(b2), n, T, C_, c3.n_out,
                                           c3.dilation, float(self.res_scale), stream_ptr()))
            return out
        # two launches through an [n, T, Cs] temporary; with tensor_cores set, the wide shapes of the upsampler
        # Conditioner (multiples of 64 channels, one above 64) run both on the wgmma kernel (jk_conv1d_tc_wide)
        h = c3(x, relu_in=True)
        return c1(h, relu_in=True, res=x, scale=self.res_scale)


class Resnet1D(nn.Module):
    def __init__(self, n_in, n_depth, m_conv=1.0, dilation_growth_rate=1, dilation_cycle=None, zero_out=False,
                 res_scale=False, reverse_dilation=False, checkpoint_res=False):
        super().__init__()
        cyc = (lambda d: d) if dilation_cycle is None else (lambda d: d % dilation_cycle)
        blocks = [ResConv1DBlock(n_in, int(m_conv * n_in), dilation=dilation_growth_rate ** cyc(d),
                                 zero_out=zero_out, res_scale=1.0 if not res_scale else 1.0 / math.sqrt(n_depth))
                  for d in range(n_depth)]
        if reverse_dilation:
            blocks = blocks[::-1]
        self.checkpoint_res = checkpoint_res
        # the reference registers the same blocks under `blocks` when gradient checkpointing is
        # requested and under `model` otherwise; checkpoints depend on it (make_models.py:124-128)
        if checkpoint_res == 1:
            self.blocks = nn.ModuleList(blocks)
        else:
            self.model = nn.Sequential(*blocks)

    def forward(self, x):
        for blk in (self.blocks if self.checkpoint_res == 1 else self.model):
            x = blk(x)
        return x


def use_tensor_cores(module, on=True):
    """switch every ResConv1DBlock and channels-last conv below `module` to the split-precision tensor-core kernels
    (jk_resblock_tc, jk_conv1d_cl with tensor_cores = 1, jk_conv1d_tc_wide) - decoder-side stacks only"""
    for m in module.modules():
        if hasattr(m, "tensor_cores"):
            m.tensor_cores = bool(on)
    return module
