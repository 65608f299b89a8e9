"""Log-probabilities of given tokens under an x_out head, straight from the activations (csrc/score.cu,
jk_xout_logprob): the [M, bins] logits are never materialised.  Used by ConditionalAutoregressive2D.logprob,
SimplePrior.score and the prefilled positions of sample(get_logprobs=True)."""
import ctypes as C

import torch as t

from ._lib import lib, check, ptr, stream_ptr


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
