"""Log-probabilities of given tokens under an x_out head, straight from the activations (csrc/score.cu,
jk_xout_logprob): the [M, bins] logits are never materialised.  Used by ConditionalAutoregressive2D.logprob,
SimplePrior.score and the prefilled positions of sample(get_logprobs=True).  xout_stats (jk_xout_stats) adds the
entropy and the most likely tokens of each row, for token_stats and sample.song_token_stats."""
import ctypes as C
from collections import namedtuple

import torch as t

from ._lib import lib, check, ptr, stream_ptr, JK_XOUT_STATS_MAX_K


def split_x_out(weight):
    """x_out [bins, W] in the hi / lo fp16 layout the kernel streams, packed once per weight load: the packed copy is
    kept on the parameter and re-made when its storage or version changes"""
    key = (weight.data_ptr(), weight._version, tuple(weight.shape), str(weight.device))
    cached = getattr(weight, "_jk_xout_split", None)
    if cached is not None and cached[0] == key:
        return cached[1]
    bins, W = weight.shape
    nbytes = C.c_size_t(0)
    check(lib().jk_xout_split_bytes(bins, W, C.byref(nbytes)))
    split = t.empty(nbytes.value, dtype=t.uint8, device=weight.device)
    w32 = weight.detach().float().contiguous()
    check(lib().jk_pack_xout_split(ptr(w32), ptr(split), bins, W, stream_ptr()))
    weight._jk_xout_split = (key, split)
    return split


def xout_logprob(h, weight, targets, get_lse=False):
    """log_softmax(h . weight^T)[m, targets[m]] in fp32 nats for every row m, and log-sum-exp of the row with get_lse.
    h: fp32 CUDA [M, W]; weight: x_out [bins, W]; targets: int64 [M]."""
    assert h.dim() == 2 and targets.shape == (h.shape[0],)
    h = h.float().contiguous()
    targets = targets.long().contiguous()
    M, W = h.shape
    bins = weight.shape[0]
    assert weight.shape[1] == W, f"x_out {tuple(weight.shape)} does not take width {W}"
    if M == 0:
        e = t.empty(0, dtype=t.float32, device=h.device)
        return (e, e.clone()) if get_lse else e
    split = split_x_out(weight)
    nbytes = C.c_size_t(0)
    check(lib().jk_xout_logprob_workspace_bytes(M, W, bins, C.byref(nbytes)))
    ws = t.empty(nbytes.value, dtype=t.uint8, device=h.device)
    logp = t.empty(M, dtype=t.float32, device=h.device)
    lse = t.empty(M, dtype=t.float32, device=h.device) if get_lse else None
    check(lib().jk_xout_logprob(ptr(h), M, W, ptr(split), bins, ptr(targets), ptr(logp), ptr(lse), ptr(ws),
                                nbytes.value, stream_ptr()))
    return (logp, lse) if get_lse else logp


TokenStats = namedtuple("TokenStats", "logp entropy topk_ids topk_logp lse")
TokenStats.__doc__ = """per-row statistics of softmax(z): logp [M] at the targets, entropy [M] in nats, topk_ids int64 [M, k]
(descending logit, ties to the lower id), topk_logp [M, k], lse [M]; a field that was not asked for is None"""


def xout_stats(h, weight, targets=None, top_k=0):
    """Entropy, the top_k most likely ids with their log-probabilities, log-sum-exp and - with targets - the
    log-probability of the targets under softmax(h . weight^T), from one fused kernel (jk_xout_stats): logp and lse are
    xout_logprob's bit for bit.  h: fp32 CUDA [M, W]; weight: x_out [bins, W]; targets: int64 [M] or None."""
    assert h.dim() == 2
    h = h.float().contiguous()
    M, W = h.shape
    bins = weight.shape[0]
    assert weight.shape[1] == W, f"x_out {tuple(weight.shape)} does not take width {W}"
    assert 0 <= top_k <= min(JK_XOUT_STATS_MAX_K, bins), f"top_k {top_k} outside [0, {min(JK_XOUT_STATS_MAX_K, bins)}]"
    if targets is not None:
        assert targets.shape == (M,)
        targets = targets.long().contiguous()
    dev = h.device
    f32 = lambda *s: t.empty(*s, dtype=t.float32, device=dev)
    out = TokenStats(logp=None if targets is None else f32(M), entropy=f32(M),
                     topk_ids=t.empty(M, top_k, dtype=t.long, device=dev) if top_k else None,
                     topk_logp=f32(M, top_k) if top_k else None, lse=f32(M))
    if M == 0:
        return out
    split = split_x_out(weight)
    nbytes = C.c_size_t(0)
    check(lib().jk_xout_stats_workspace_bytes(M, W, bins, top_k, C.byref(nbytes)))
    ws = t.empty(nbytes.value, dtype=t.uint8, device=dev)
    check(lib().jk_xout_stats(ptr(h), M, W, ptr(split), bins, ptr(targets), top_k, ptr(out.logp), ptr(out.entropy),
                              ptr(out.topk_ids), ptr(out.topk_logp), ptr(out.lse), ptr(ws), nbytes.value, stream_ptr()))
    return out
