"""Lyric alignment from attention weights (reference jukebox/align.py:15-84).

For every window ("hop") of the top-level codes the prior's forward pass is run with attention recording on the model's
designated alignment layer; the chosen head's [codes x lyric tokens] weights of each hop are scattered back to the columns
of the full lyric (the labeller tells which full-lyric index each of the window's n_tokens slots came from) and later hops
are overwritten by earlier ones, exactly as the reference's reversed loop does.

The forward pass is SimplePrior.z_forward with the sampling fp16 flag, as in the reference (sample.py:118-119 ->
get_alignment):
  fp16=True  - the fp16 prefill records the layer's weights on the tensor cores (csrc/prefill.cu, fp16 weights, the
               reference's fp16 mode); as many items per call as one prefill takes (items_per_prefill of the prior's
               autoregressive model), since prefill rows are independent and the weights are the same bits as item by
               item; an engine built for fewer items is rebuilt once, on the first window, and serves every later one.
               A window longer than the prefill capacity (JK_PREFILL_MAX) records on the fp32 path instead;
  fp16=False - the fp32 forward-mode path (Transformer.forward(sample=False) -> csrc/f32_path.cu), item by item.
"""
import numpy as np
import torch as t

from .utils.sample_utils import get_starts


def pad_to_context(z, n_ctx):
    """codes shorter than one context are right-padded with code 0; returns (z, pad)"""
    pad = max(0, n_ctx - z.shape[1])
    if pad:
        z = t.cat([z, t.zeros(z.shape[0], pad, dtype=z.dtype, device=z.device)], dim=1)
    return z, pad


def hop_weights(prior, z_window, y, fp16):
    """[bs, n_ctx, n_tokens] weights (fp32 array) of the alignment head for one window; each z_forward call records a
    [items, heads, n_ctx, keys] tensor: in fp16 as many items as one prefill takes (item by item when the prior has no
    prefill), in fp32 one, like the reference"""
    layer, head = prior.alignment_layer, prior.alignment_head
    rows = []
    bs = z_window.shape[0]
    step = (prior.prior.items_per_prefill(bs) or 1) if fp16 and bs > 1 else 1
    for i in range(0, bs, step):
        ws = prior.z_forward(z_window[i:i + step], [], y[i:i + step], fp16=fp16, get_attn_weights={layer})
        assert len(ws) == 1
        rows.append(ws[0][:, head].float())
    w = t.cat(rows, dim=0)
    assert w.shape == (z_window.shape[0], prior.n_ctx, prior.n_tokens), tuple(w.shape)
    return w.cpu().numpy()


def stitch(hops, indices, starts, full_lengths, total_length, n_ctx, pad):
    """hops[start]: [bs, n_ctx, n_tokens]; indices[start][item]: full-lyric column of each token slot.
    -> per item [total_length - pad, len(full lyric)]"""
    out = []
    for item, n_full in enumerate(full_lengths):
        a = np.zeros((total_length, n_full + 1))
        for start in reversed(starts):
            a[start:start + n_ctx, indices[start][item]] = hops[start][item]
        out.append(a[:total_length - pad, :-1])      # drop the padding rows and the column of the "no token" slot
    return out


def get_alignment(x, zs, labels, prior, fp16, hps):
    """alignments: list (one per item) of [codes, lyric characters] attention maps - signature of the reference"""
    level = hps.levels - 1
    n_ctx, n_tokens = prior.n_ctx, prior.n_tokens
    z, pad = pad_to_context(zs[level], n_ctx)
    bs, total_length = z.shape
    hop = int(hps.hop_fraction[level] * n_ctx)
    starts = list(get_starts(total_length, n_ctx, hop))
    hops, indices = {}, {}
    with t.no_grad():
        for start in starts:
            y, idx = prior.get_y(labels, start, get_indices=True)
            assert len(idx) == bs and all(len(i) == n_tokens for i in idx)
            hops[start] = hop_weights(prior, z[:, start:start + n_ctx], y, fp16)
            indices[start] = idx
    full_lengths = [len(info['full_tokens']) for info in labels['info']]
    return stitch(hops, indices, starts, full_lengths, total_length, n_ctx, pad)
