"""Codebook quantise / dequantise (reference: jukebox/vqvae/bottleneck.py:88-147, 181-215).

The sampling-time surface (encode / decode) and the evaluation-mode forward, which VQVAE.forward uses to measure a
model: quantise, dequantise, commit loss, no codebook update.  Tensors are channels-last [N, T, emb_width] (the
reference's are NCT).  The k-means EMA updates (`update_k=True`, a Bottleneck in training mode) are training and out of
scope."""
import torch as t
import torch.nn as nn

from .._lib import lib, check, ptr, stream_ptr


class BottleneckBlock(nn.Module):
    def __init__(self, k_bins, emb_width, mu):
        super().__init__()
        self.k_bins, self.emb_width, self.mu = k_bins, emb_width, mu
        self.register_buffer('k', t.zeros(k_bins, emb_width))
        self.threshold = 1.0

    def quantise(self, x):
        """x: [M, emb_width] fp32 -> (int64 [M], fp32 [M] min distance)"""
        x = x.float().contiguous()
        idx = t.empty(x.shape[0], dtype=t.int64, device=x.device)
        dist = t.empty(x.shape[0], dtype=t.float32, device=x.device)
        if x.shape[0] == 0:
            if not x.is_cuda:
                raise RuntimeError("jukebox_b200 kernels need CUDA tensors (no CPU fallback)")
            return idx, dist
        check(lib().jk_vq_argmin(ptr(x), ptr(self.k.float().contiguous()), ptr(idx), ptr(dist), x.shape[0],
                                 self.k_bins, self.emb_width, stream_ptr()))
        return idx, dist

    def dequantise(self, x_l):
        x_l = x_l.contiguous().view(-1).long()
        out = t.empty(x_l.shape[0], self.emb_width, dtype=t.float32, device=x_l.device)
        if x_l.shape[0] == 0:
            return out
        check(lib().jk_vq_gather(ptr(x_l), ptr(self.k.float().contiguous()), ptr(out), x_l.shape[0], self.k_bins,
                                 self.emb_width, stream_ptr()))
        return out

    def encode(self, x):
        """x: [N, T, emb_width] channels-last -> codes [N, T]"""
        N, T, w = x.shape
        assert w == self.emb_width, f"Expected {w} to be {self.emb_width}"
        x_l, _ = self.quantise(x.reshape(N * T, w))
        return x_l.view(N, T)

    def decode(self, x_l):
        N, T = x_l.shape
        return self.dequantise(x_l).view(N, T, self.emb_width)

    def forward(self, x, update_k=False):
        """x: [N, T, emb_width] -> (codes [N, T], decoder input [N, T, emb_width], commit_loss, dict(fit, pn))
        (bottleneck.py:168-193 with update_k False)"""
        if update_k:
            raise NotImplementedError("codebook EMA training is out of scope (SURVEY.md section 2.1 #4)")
        N, T, w = x.shape
        assert w == self.emb_width, f"Expected {w} to be {self.emb_width}"
        x = x.float().reshape(N * T, w)
        prenorm = t.norm(x - t.mean(x)) / x.numel() ** 0.5
        x_l, min_distance = self.quantise(x)
        fit = t.mean(min_distance)
        x_d = self.dequantise(x_l)
        commit_loss = t.norm(x_d - x) ** 2 / x.numel()
        x_d = x + (x_d - x)          # the reference's straight-through form, same rounding
        return x_l.view(N, T), x_d.view(N, T, w), commit_loss, dict(fit=fit, pn=prenorm)


class Bottleneck(nn.Module):
    def __init__(self, l_bins, emb_width, mu, levels):
        super().__init__()
        self.levels = levels
        self.level_blocks = nn.ModuleList(BottleneckBlock(l_bins, emb_width, mu) for _ in range(levels))

    def encode(self, xs):
        return [blk.encode(x) for blk, x in zip(self.level_blocks, xs)]

    def decode(self, zs, start_level=0, end_level=None):
        if end_level is None:
            end_level = self.levels
        return [blk.decode(z) for blk, z in zip(self.level_blocks[start_level:end_level], zs)]

    def forward(self, xs):
        """evaluation mode only (bottleneck.py:200-215 with self.training False): no codebook update and, as in the
        reference, no per-level metrics"""
        zs, xs_quantised, commit_losses = [], [], []
        for blk, x in zip(self.level_blocks, xs):
            z, x_quantised, commit_loss, _ = blk(x, update_k=self.training)
            zs.append(z)
            xs_quantised.append(x_quantised.detach())
            commit_losses.append(commit_loss)
        return zs, xs_quantised, commit_losses, []
