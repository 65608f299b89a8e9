"""TEST INFRASTRUCTURE - fp64 numpy restatement of token scoring, used only by tests/.

Reference: the loss of jukebox/prior/autoregressive.py forward (F.cross_entropy of x_out(acts) against the tokens,
divided by ln 2 for bits) taken per token instead of averaged: logp[m] = log_softmax(z[m])[target[m]].  It checks
jk_xout_logprob (z = h . w^T from the activations) and jk_sample_categorical_scored (z given).
"""
import numpy as np


def logsumexp(z):
    """log sum exp over the last axis, fp64"""
    z = np.asarray(z, np.float64)
    mx = z.max(-1, keepdims=True)
    return (mx + np.log(np.exp(z - mx).sum(-1, keepdims=True)))[..., 0]


def logprob_from_logits(z, targets):
    """log_softmax(z)[..., target] in fp64: z [..., bins], targets [...] -> [...]"""
    z = np.asarray(z, np.float64)
    t = np.asarray(targets, np.int64)
    return np.take_along_axis(z, t[..., None], -1)[..., 0] - logsumexp(z)


def xout_logprob(h, w, targets):
    """(logp, lse) of z = h . w^T in fp64: h [M, W], w [bins, W] (nn.Linear layout), targets [M]"""
    z = np.asarray(h, np.float64) @ np.asarray(w, np.float64).T
    return logprob_from_logits(z, targets), logsumexp(z)


def bits_per_token(logp):
    """-logp / ln 2 averaged over the last axis (per item)"""
    return -np.asarray(logp, np.float64).mean(-1) / np.log(2.0)
