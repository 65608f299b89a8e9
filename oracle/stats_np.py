"""TEST INFRASTRUCTURE - fp64 numpy restatement of per-token statistics of the predictive distribution, used only by
tests/.

The reference computes the distribution as softmax(x_out(acts)) (jukebox/prior/autoregressive.py) and samples from it;
these are the standard statistics of that distribution at each position: its entropy H = -sum p log p, and its k most
likely tokens (torch.topk of the log-softmax, ties to the lower id).  They check jk_xout_stats.  Log-probability and
log-sum-exp come from oracle/score_np.py.
"""
import numpy as np

from .score_np import logsumexp, logprob_from_logits


def entropy_from_logits(z):
    """H = -sum p log p of softmax(z) over the last axis, fp64"""
    z = np.asarray(z, np.float64)
    lp = z - logsumexp(z)[..., None]
    return -(np.exp(lp) * lp).sum(-1)


def topk_from_logits(z, k):
    """the k largest logits of the last axis by descending value, ties to the lower id: (ids int64, log_softmax there)"""
    z = np.asarray(z, np.float64)
    ids = np.argsort(-z, axis=-1, kind="stable")[..., :k]
    return ids.astype(np.int64), np.take_along_axis(z, ids, -1) - logsumexp(z)[..., None]


def xout_stats(h, w, targets=None, k=0):
    """(logp or None, entropy, topk_ids, topk_logp, lse, z) of z = h . w^T in fp64: h [M, W], w [bins, W]"""
    z = np.asarray(h, np.float64) @ np.asarray(w, np.float64).T
    ids, tlp = topk_from_logits(z, k)
    lp = None if targets is None else logprob_from_logits(z, targets)
    return lp, entropy_from_logits(z), ids, tlp, logsumexp(z), z
