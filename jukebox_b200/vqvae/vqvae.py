"""VQVAE.encode / decode and the evaluation-mode forward on the GPU (reference: jukebox/vqvae/vqvae.py:21-228).

Audio stays [N, T, 1] (the reference permutes to NCT for cuDNN; here every tensor is
channels-last, which is what the kernels want, so preprocess/postprocess are no-ops)."""
import numpy as np
import torch as t
import torch.nn as nn

from .encdec import Encoder, Decoder
from .bottleneck import Bottleneck
from ..utils.audio_utils import (DefaultSTFTValues, audio_postprocess, convergence, multispectral_loss, stft_stats)


def calculate_strides(strides, downs):
    return [stride ** down for stride, down in zip(strides, downs)]


def _loss_fn(loss_fn, x_target, x_pred, hps):
    """Reconstruction loss of vqvae.py:21-40, scaled by the dataset's bandwidth: 'l1', 'l2', 'linf' (mean of the
    hps.linf_k largest squared errors per clip) or 'lmix' (their hps.lmix_* weighted sum, zero weights skipped)."""
    err = x_pred - x_target
    if loss_fn == 'l1':
        return err.abs().mean() / hps.bandwidth['l1']
    if loss_fn == 'l2':
        return err.square().mean() / hps.bandwidth['l2']
    if loss_fn == 'linf':
        worst = t.topk(err.square().reshape(x_target.shape[0], -1), hps.linf_k, dim=1).values
        return worst.mean() / hps.bandwidth['l2']
    if loss_fn == 'lmix':
        total = 0.0
        for name, weight in (('l1', hps.lmix_l1), ('l2', hps.lmix_l2), ('linf', hps.lmix_linf)):
            if weight:
                total = total + weight * _loss_fn(name, x_target, x_pred, hps)
        return total
    raise ValueError(f"Unknown loss_fn {loss_fn}")


class VQVAE(nn.Module):
    def __init__(self, input_shape, levels, downs_t, strides_t, emb_width, l_bins, mu, commit, spectral,
                 multispectral, multipliers=None, use_bottleneck=True, **block_kwargs):
        super().__init__()
        assert use_bottleneck, "NoBottleneck variants are training-only experiments"
        self.sample_length = input_shape[0]
        x_shape, x_channels = input_shape[:-1], input_shape[-1]
        self.x_shape = x_shape
        self.downsamples = calculate_strides(strides_t, downs_t)
        self.hop_lengths = np.cumprod(self.downsamples)
        self.z_shapes = [(x_shape[0] // self.hop_lengths[level],) for level in range(levels)]
        self.levels = levels
        self.multipliers = [1] * levels if multipliers is None else multipliers
        assert len(self.multipliers) == levels, "Invalid number of multipliers"

        def kw(level):
            d = dict(block_kwargs)
            d["width"] *= self.multipliers[level]
            d["depth"] *= self.multipliers[level]
            return d
        self.encoders = nn.ModuleList(Encoder(x_channels, emb_width, level + 1, downs_t[:level + 1],
                                              strides_t[:level + 1], **kw(level)) for level in range(levels))
        self.decoders = nn.ModuleList(Decoder(x_channels, emb_width, level + 1, downs_t[:level + 1],
                                              strides_t[:level + 1], **kw(level)) for level in range(levels))
        self.bottleneck = Bottleneck(l_bins, emb_width, mu, levels)
        self.downs_t, self.strides_t, self.l_bins = downs_t, strides_t, l_bins
        self.commit, self.spectral, self.multispectral = commit, spectral, multispectral

    def preprocess(self, x):
        assert len(x.shape) == 3
        return x.float()

    def postprocess(self, x):
        return x

    def _decode(self, zs, start_level=0, end_level=None):
        if end_level is None:
            end_level = self.levels
        assert len(zs) == end_level - start_level
        xs_quantised = self.bottleneck.decode(zs, start_level=start_level, end_level=end_level)
        decoder, x_quantised = self.decoders[start_level], xs_quantised[0:1]
        return self.postprocess(decoder(x_quantised, all_levels=False))

    def decode(self, zs, start_level=0, end_level=None, bs_chunks=1):
        z_chunks = [t.chunk(z, bs_chunks, dim=0) for z in zs]
        x_outs = [self._decode([zc[i] for zc in z_chunks], start_level=start_level, end_level=end_level)
                  for i in range(bs_chunks)]
        return t.cat(x_outs, dim=0)

    def _encode(self, x, start_level=0, end_level=None):
        if end_level is None:
            end_level = self.levels
        x_in = self.preprocess(x)
        xs = [self.encoders[level](x_in)[-1] for level in range(self.levels)]
        return self.bottleneck.encode(xs)[start_level:end_level]

    def encode(self, x, start_level=0, end_level=None, bs_chunks=1):
        zs_list = [self._encode(x_i, start_level=start_level, end_level=end_level)
                   for x_i in t.chunk(x, bs_chunks, dim=0)]
        return [t.cat(z, dim=0) for z in zip(*zs_list)]

    def sample(self, n_samples):
        dev = self.bottleneck.level_blocks[0].k.device
        zs = [t.randint(0, self.l_bins, size=(n_samples, *z_shape), device=dev) for z_shape in self.z_shapes]
        return self.decode(zs)

    def forward(self, x, hps, loss_fn='l1'):
        """Evaluation of a reconstruction (vqvae.py:150-228 in eval mode): x [N, T, 1] -> (level-0 reconstruction,
        loss, metrics).  Every level encodes, quantises and decodes its own codes; the metrics are the reference's
        eval-mode keys, each a detached 0-dim tensor.  hps needs the reference's loss settings and `bandwidth`,
        dict(l1, l2, spec) of the dataset (train.py computes it with calculate_bandwidth)."""
        if self.training:
            raise NotImplementedError("VQ-VAE training (codebook EMA, gradients) is out of scope: call .eval() first")
        try:
            bandwidth = hps.bandwidth
        except (AttributeError, KeyError):
            bandwidth = None
        if not isinstance(bandwidth, dict) or not {'l1', 'l2', 'spec'} <= set(bandwidth):
            raise ValueError("hps.bandwidth must be dict(l1, l2, spec), the dataset statistics the losses are scaled by")
        with t.no_grad():
            return self._forward(x, hps, loss_fn)

    def _forward(self, x, hps, loss_fn):
        metrics = {}
        x_in = self.preprocess(x)
        xs = [self.encoders[level](x_in)[-1] for level in range(self.levels)]
        zs, xs_quantised, commit_losses, _ = self.bottleneck(xs)
        x_outs = []
        for level in range(self.levels):
            x_out = self.decoders[level](xs_quantised[level:level + 1], all_levels=False)
            assert x_out.shape == x_in.shape, (tuple(x_out.shape), tuple(x_in.shape))
            x_outs.append(x_out)

        recons_loss = t.zeros((), device=x.device)
        spec_loss = t.zeros((), device=x.device)
        multispec_loss = t.zeros((), device=x.device)
        x_target = audio_postprocess(x.float(), hps)
        for level in reversed(range(self.levels)):
            x_out = audio_postprocess(self.postprocess(x_outs[level]), hps)
            this_recons_loss = _loss_fn(loss_fn, x_target, x_out, hps)
            # the default config's norms; at level 0 they also give the spectral convergence metric below
            residual_norm, gt_norm = stft_stats(x_target, x_out, DefaultSTFTValues(hps))
            if hps.use_nonrelative_specloss:
                this_spec_loss = t.mean(residual_norm / hps.bandwidth['spec'])
            else:
                this_spec_loss = t.mean(convergence(residual_norm, gt_norm))
            this_multispec_loss = t.mean(multispectral_loss(x_target, x_out, hps) / hps.bandwidth['spec'])
            metrics[f'recons_loss_l{level + 1}'] = this_recons_loss
            metrics[f'spectral_loss_l{level + 1}'] = this_spec_loss
            metrics[f'multispectral_loss_l{level + 1}'] = this_multispec_loss
            recons_loss += this_recons_loss
            spec_loss += this_spec_loss
            multispec_loss += this_multispec_loss

        commit_loss = sum(commit_losses)
        loss = recons_loss + self.spectral * spec_loss + self.multispectral * multispec_loss + self.commit * commit_loss

        # x_out, residual_norm and gt_norm are level 0's, left over from the reversed loop as in the reference
        sc = t.mean(convergence(residual_norm, gt_norm))
        l2_loss = _loss_fn("l2", x_target, x_out, hps)
        l1_loss = _loss_fn("l1", x_target, x_out, hps)
        linf_loss = _loss_fn("linf", x_target, x_out, hps)
        metrics.update(dict(recons_loss=recons_loss, spectral_loss=spec_loss, multispectral_loss=multispec_loss,
                            spectral_convergence=sc, l2_loss=l2_loss, l1_loss=l1_loss, linf_loss=linf_loss,
                            commit_loss=commit_loss))
        for key, val in metrics.items():
            metrics[key] = val.detach()
        return x_out, loss, metrics
