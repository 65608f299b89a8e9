"""Parameter containers with the reference's names (jukebox/transformer/ops.py) and the
logit post-processing that stays in torch.

Conv1D / LayerNorm here do NOT compute: at sampling time their parameters are packed into the
decode engine (jukebox_b200/engine.py) and all arithmetic happens in libjkb200.so.
"""
import torch as t
import torch.nn as nn
import torch.nn.functional as F


class LayerNorm(nn.Module):
    """weight/bias holder for the fused LayerNorm (reference: ops.py:14-24, eps 1e-5)."""

    def __init__(self, normalized_shape, eps=1e-5):
        super().__init__()
        self.normalized_shape = (int(normalized_shape),)
        self.eps = eps
        self.weight = nn.Parameter(t.ones(normalized_shape))
        self.bias = nn.Parameter(t.zeros(normalized_shape))

    def forward(self, x):
        """fp32 rows on the GPU through jk_layernorm_f32 (used by the Conditioner)."""
        from .._lib import lib, check, ptr, stream_ptr
        x = x.float().contiguous()
        y = t.empty_like(x)
        rows = x.numel() // x.shape[-1]
        check(lib().jk_layernorm_f32(ptr(x), ptr(self.weight.detach().float().contiguous()),
                                     ptr(self.bias.detach().float().contiguous()), ptr(y), rows,
                                     x.shape[-1], self.eps, stream_ptr()))
        return y


class Conv1D(nn.Module):
    """w: [n_in, n_out] (transposed w.r.t. nn.Linear), b: [n_out]  - reference ops.py:83-96."""

    def __init__(self, n_in, n_out, zero_out=False, init_scale=1.0):
        super().__init__()
        self.n_in, self.n_out = n_in, n_out
        w = t.zeros(n_in, n_out) if zero_out else t.empty(n_in, n_out).normal_(std=0.02 * init_scale)
        self.w = nn.Parameter(w)
        self.b = nn.Parameter(t.zeros(n_out))

    def forward(self, x):
        raise RuntimeError("Conv1D is a parameter container; it runs inside the decode engine "
                           "(Transformer.forward(sample=True)). No eager path exists.")


def _convert_conv_weights_to_fp16(l):
    if isinstance(l, Conv1D):
        l.w.data = l.w.data.half()


def _convert_conv_weights_to_fp32(l):
    if isinstance(l, Conv1D):
        l.w.data = l.w.data.float()


def filter_logits(logits, top_k=0, top_p=0.0, filter_value=-float('Inf')):
    """top-k / nucleus filtering of a logits tensor as a torch expression, semantics of the reference's
    ops.py:113-142.  The sampling loop uses the one-launch `filter_logits_scaled` below; this form stays for
    callers that hold arbitrary-shaped logits and as the checker of that kernel in the GPU tests."""
    out = logits.clone()
    top_k = min(top_k, out.size(-1))
    assert (top_k == 0) or (top_p == 0.0)
    if top_k > 0:
        kth = t.topk(out, top_k, dim=-1)[0][..., -1:]
        out[out < kth] = filter_value
    if top_p > 0.0:
        srt, order = t.sort(out, descending=True, dim=-1)
        cum = t.cumsum(F.softmax(srt, dim=-1), dim=-1)
        drop = cum > top_p
        drop[..., 1:] = drop[..., :-1].clone()
        drop[..., 0] = 0
        mask = t.zeros_like(out, dtype=t.bool).scatter_(dim=-1, index=order, src=drop)
        out[mask] = filter_value
    return out


def filter_logits_scaled(logits, temp, top_k, top_p, out=None):
    """filter_logits(logits / temp, top_k, top_p) in ONE launch (jk_filter_logits): the sampling loop's
    `x = x / temp; x = filter_logits(x, top_k, top_p)` (reference autoregressive.py:232-234).  logits: fp32 CUDA [N, bins]
    with unit inner stride; returns fp32 [N, bins] (written into `out` when given)."""
    from .._lib import lib, check, stream_ptr
    import ctypes as C
    assert logits.dtype == t.float32 and logits.dim() == 2 and logits.stride(1) == 1
    if not logits.is_cuda:
        raise RuntimeError("filter_logits_scaled needs CUDA tensors (no CPU path)")
    if out is None:
        out = t.empty(logits.shape, dtype=t.float32, device=logits.device)
    assert out.shape == logits.shape and out.dtype == t.float32 and out.stride(1) == 1
    check(lib().jk_filter_logits(C.c_void_p(logits.data_ptr()), logits.stride(0), logits.shape[0], logits.shape[1],
                                 float(temp), int(top_k), float(top_p), C.c_void_p(out.data_ptr()), out.stride(0),
                                 stream_ptr()))
    return out


def sample_categorical(logits, temp, seed, position, tokens):
    """tokens[:, position] ~ Categorical(logits = logits / temp) in one launch (jk_sample_categorical;
    reference autoregressive.py:233-235).  logits: fp32 CUDA [N, bins] view with unit inner stride,
    tokens: int64 CUDA [N, L].  (seed, position, row) fixes the uniform behind each draw."""
    from .._lib import lib, check, ptr, stream_ptr
    assert logits.dtype == t.float32 and logits.dim() == 2 and logits.stride(1) == 1
    assert tokens.dtype == t.int64 and tokens.dim() == 2 and tokens.stride(1) == 1
    if not logits.is_cuda or not tokens.is_cuda:
        raise RuntimeError("sample_categorical needs CUDA tensors (no CPU path)")
    import ctypes as C
    check(lib().jk_sample_categorical(C.c_void_p(logits.data_ptr()), logits.stride(0), logits.shape[0],
                                      logits.shape[1], float(temp), C.c_uint64(seed & (2 ** 64 - 1)), int(position),
                                      C.c_void_p(tokens.data_ptr()), tokens.stride(0), stream_ptr()))


def sample_categorical_scored(logits, raw, temp, seed, position, tokens, logp):
    """sample_categorical(logits, temp, seed, position, tokens) - the same token - and, in the same launch,
    logp[:, position] = log_softmax(raw)[token] (jk_sample_categorical_scored).  raw: the unfiltered logits the draw
    came from (temperature 1).  logits=None draws nothing and scores the given tokens[:, position].
    logits / raw: fp32 CUDA [N, bins] with unit inner stride; tokens int64 [N, L], logp fp32 [N, L]."""
    from .._lib import lib, check, stream_ptr
    import ctypes as C
    for x in (raw, logits):
        assert x is None or (x.dtype == t.float32 and x.dim() == 2 and x.stride(1) == 1 and x.is_cuda)
    assert tokens.dtype == t.int64 and tokens.dim() == 2 and tokens.stride(1) == 1
    assert logp.dtype == t.float32 and logp.dim() == 2 and logp.stride(1) == 1
    if not tokens.is_cuda or not logp.is_cuda:
        raise RuntimeError("sample_categorical_scored needs CUDA tensors (no CPU path)")
    lp = C.c_void_p(0 if logits is None else logits.data_ptr())
    check(lib().jk_sample_categorical_scored(lp, 0 if logits is None else logits.stride(0), C.c_void_p(raw.data_ptr()),
                                             raw.stride(0), raw.shape[0], raw.shape[1], float(temp),
                                             C.c_uint64(seed & (2 ** 64 - 1)), int(position),
                                             C.c_void_p(tokens.data_ptr()), tokens.stride(0),
                                             C.c_void_p(logp.data_ptr()), logp.stride(0), stream_ptr()))


def sample_guided(c, u, s, temp, top_k, top_p, seed, position, tokens, tokens_alt, logp=None):
    """One guided draw per pair in one launch (jk_sample_guided): g = c + s * (c - u), then filter_logits_scaled(g, temp,
    top_k, top_p) when a filter is set and the draw of sample_categorical - the same token, written to both
    tokens[:, position] and tokens_alt[:, position].  With logp: logp[:, position] = log_softmax(c)[token], the
    conditional likelihood at temperature 1.  c / u: fp32 CUDA [n, bins] with unit inner stride; tokens / tokens_alt
    int64 [n, L]; logp fp32 [n, L]."""
    from .._lib import lib, check, stream_ptr
    import ctypes as C
    for x in (c, u):
        assert x.dtype == t.float32 and x.dim() == 2 and x.stride(1) == 1 and x.is_cuda
    assert c.shape == u.shape
    for x in (tokens, tokens_alt):
        assert x.dtype == t.int64 and x.dim() == 2 and x.stride(1) == 1 and x.is_cuda and x.shape[0] == c.shape[0]
    if logp is not None:
        assert logp.dtype == t.float32 and logp.dim() == 2 and logp.stride(1) == 1 and logp.is_cuda
    vp = lambda x: C.c_void_p(0 if x is None else x.data_ptr())
    check(lib().jk_sample_guided(vp(c), c.stride(0), vp(u), u.stride(0), c.shape[0], c.shape[1], float(s), float(temp),
                                 int(top_k), float(top_p), C.c_uint64(seed & (2 ** 64 - 1)), int(position), vp(tokens),
                                 tokens.stride(0), vp(tokens_alt), tokens_alt.stride(0),
                                 vp(None if logp is None else c), vp(logp), 0 if logp is None else logp.stride(0),
                                 stream_ptr()))
