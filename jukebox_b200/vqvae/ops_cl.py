"""Channels-last ([N, T, C] fp32) convolution leaves for the VQ-VAE and the upsampler
Conditioner.  Parameters keep torch's names and shapes (`weight` [O, C, K] / [C, O, K], `bias`)
so reference checkpoints load strictly; the arithmetic is libjkb200's jk_conv1d_cl, and jk_conv1d_tc_wide for the
Conditioner's wide decoder-side convs when `tensor_cores` is set.
"""
import ctypes as C

import torch as t
import torch.nn as nn

from .. import _lib
from .._lib import lib, check, ptr, stream_ptr


def _wide_tc(x, c_out, taps, in_stride, tensors):
    """the shapes jk_conv1d_tc_wide takes (jkb200.h): channels multiples of 64 with one above 64, stride-1 input,
    <= 3 taps, >= 128 input positions, 16-byte aligned tensors"""
    _, t_in, c_in = x.shape
    return (c_in % 64 == 0 and c_out % 64 == 0 and max(c_in, c_out) > 64 and in_stride == 1 and len(taps) <= 3
            and t_in >= 128 and all(v is None or v.data_ptr() % 16 == 0 for v in tensors))


def _split(w_packed):
    """packed fp32 [k, c_in, c_out] -> the hi / lo fp16 layout jk_conv1d_tc_wide streams (uint8 bytes)"""
    k, c_in, c_out = w_packed.shape
    nbytes = C.c_size_t(0)
    check(lib().jk_conv_weight_split_bytes(k, c_in, c_out, C.byref(nbytes)))
    s = t.empty(nbytes.value, dtype=t.uint8, device=w_packed.device)
    check(lib().jk_pack_conv_weight_split(ptr(w_packed), ptr(s), k, c_in, c_out, stream_ptr()))
    return s


def _conv(x, w_packed, bias, t_out, c_out, taps, in_stride=1, out=None, out_stride=1, out_offset=0,
          relu_in=False, scale=1.0, res=None, tensor_cores=False, split=None):
    """`split` (tensor_cores only): a callable returning the split weight, called when the shape takes the wide
    tensor-core kernel"""
    assert x.dim() == 3 and x.dtype == t.float32
    x = x.contiguous()
    n, t_in, c_in = x.shape
    if out is None:
        out = t.empty(n, t_out * out_stride, c_out, dtype=t.float32, device=x.device)
    wide = tensor_cores and split is not None and _wide_tc(x, c_out, taps, in_stride, (x, out, res, bias))
    a = _lib.ConvArgs()
    a.inp, a.t_in, a.c_in = ptr(x), t_in, c_in
    a.out, a.t_out, a.c_out = ptr(out), t_out, c_out
    a.w, a.bias, a.res = ptr(w_packed), ptr(bias), ptr(res)
    a.n_taps = len(taps)
    for i, o in enumerate(taps):
        a.tap_off[i] = int(o)
    a.in_stride, a.out_stride, a.out_offset = in_stride, out_stride, out_offset
    a.relu_in, a.scale, a.n = int(relu_in), float(scale), n
    a.tensor_cores = int(bool(tensor_cores))
    if wide:
        check(lib().jk_conv1d_tc_wide(C.byref(a), ptr(split()), stream_ptr()))
    else:
        check(lib().jk_conv1d_cl(C.byref(a), stream_ptr()))
    return out


class _ConvBase(nn.Module):
    transposed = False

    def __init__(self):
        super().__init__()
        self._packed = None
        self._split = None
        # decoder-side stacks set this (resnet.use_tensor_cores): split-precision tensor-core kernel, free summation order.
        # The encoder, whose output feeds the bit-exact codebook argmin, keeps the exact-FMA kernels.
        self.tensor_cores = False
        self.register_load_state_dict_post_hook(lambda m, keys: m._drop())

    def _drop(self):
        self._packed = None
        self._split = None

    def _apply(self, fn, *a, **k):
        self._drop()
        return super()._apply(fn, *a, **k)

    def packed(self):
        """[k, c_in, c_out] fp32 on the parameter's device (packed once per weight load)."""
        if self._packed is None:
            w = self.weight.detach().float().contiguous()
            if self.transposed:
                c_in, c_out, k = w.shape
            else:
                c_out, c_in, k = w.shape
            p = t.empty(k, c_in, c_out, dtype=t.float32, device=w.device)
            check(lib().jk_pack_conv_weight(ptr(w), ptr(p), c_out, c_in, k, int(self.transposed), stream_ptr()))
            self._packed = (p, self.bias.detach().float().contiguous())
        return self._packed

    def split(self):
        """the packed weight in jk_conv1d_tc_wide's hi / lo fp16 layout (split once per weight load)"""
        if self._split is None:
            self._split = _split(self.packed()[0])
        return self._split


class Conv1d(_ConvBase):
    """torch.nn.Conv1d(n_in, n_out, k, stride, padding, dilation) on channels-last tensors.
    Supported geometries are the ones the reference builds (encdec.py:17,20,35; resnet.py:33-35):
    k3 'same' dilated, k1, and k = 2*stride with padding stride//2 (stride 2)."""

    def __init__(self, n_in, n_out, kernel_size, stride=1, padding=0, dilation=1):
        super().__init__()
        self.n_in, self.n_out, self.k, self.stride, self.padding, self.dilation = n_in, n_out, kernel_size, stride, padding, dilation
        self.weight = nn.Parameter(t.empty(n_out, n_in, kernel_size))
        self.bias = nn.Parameter(t.empty(n_out))
        bound = 1.0 / (n_in * kernel_size) ** 0.5
        nn.init.uniform_(self.weight, -bound, bound)
        nn.init.uniform_(self.bias, -bound, bound)
        if stride == 1:
            assert padding == dilation * (kernel_size - 1) // 2, "only 'same' convolutions"
            self.taps = [(i - (kernel_size - 1) // 2) * dilation for i in range(kernel_size)]
        else:
            assert stride == 2 and kernel_size == 4 and padding == 1 and dilation == 1
            self.taps = [-1, 0, 1, 2]

    def forward(self, x, relu_in=False, res=None, scale=1.0):
        w, b = self.packed()
        t_out = x.shape[1] // self.stride
        return _conv(x, w, b, t_out, self.n_out, self.taps, in_stride=self.stride, relu_in=relu_in,
                     scale=scale, res=res, tensor_cores=self.tensor_cores, split=self.split)


class ConvTranspose1d(_ConvBase):
    """torch.nn.ConvTranspose1d(n_in, n_out, 4, 2, 1) (encdec.py:41): two 2-tap phases."""
    transposed = True

    def __init__(self, n_in, n_out, kernel_size, stride, padding):
        super().__init__()
        assert kernel_size == 4 and stride == 2 and padding == 1, "only k4 s2 p1 (stride_t = 2)"
        self.n_in, self.n_out = n_in, n_out
        self.weight = nn.Parameter(t.empty(n_in, n_out, kernel_size))
        self.bias = nn.Parameter(t.empty(n_out))
        bound = 1.0 / (n_out * kernel_size) ** 0.5
        nn.init.uniform_(self.weight, -bound, bound)
        nn.init.uniform_(self.bias, -bound, bound)
        self._phases = None

    def _drop(self):
        self._packed = None
        self._phases = None
        self._split = None

    def split(self):
        """the two phases' packed weights in jk_conv1d_tc_wide's hi / lo fp16 layout (split once per weight load)"""
        if self._split is None:
            self._split = tuple(_split(p) for p in self._phases)
        return self._split

    def forward(self, x):
        w, b = self.packed()
        if self._phases is None:
            # out[2m] = w1.x[m] + w3.x[m-1] ; out[2m+1] = w0.x[m+1] + w2.x[m]
            self._phases = (t.stack([w[1], w[3]]).contiguous(), t.stack([w[0], w[2]]).contiguous())
        n, T, _ = x.shape
        out = t.empty(n, 2 * T, self.n_out, dtype=t.float32, device=x.device)
        _conv(x, self._phases[0], b, T, self.n_out, [0, -1], out=out, out_stride=2, out_offset=0, tensor_cores=self.tensor_cores,
              split=lambda: self.split()[0])
        _conv(x, self._phases[1], b, T, self.n_out, [1, 0], out=out, out_stride=2, out_offset=1, tensor_cores=self.tensor_cores,
              split=lambda: self.split()[1])
        return out


class ReLU(nn.Module):
    """index placeholder inside nn.Sequential (the ReLU is fused into the following conv)."""

    def forward(self, x):
        raise RuntimeError("fused into the next convolution")
