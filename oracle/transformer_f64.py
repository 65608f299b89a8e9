"""Float64 restatement of one transformer layer, with a first-order bound on what fp32 arithmetic may add to it.

TEST INFRASTRUCTURE ONLY (only tests/ may import it).  torch, float64, on whatever device the tensors live on, so the
GPU tests can evaluate a layer at the priors' real geometry (8 576 keys, head_dim 480, 512 encoder rows) in milliseconds.

What is restated (reference file:line, under jukebox/), at the points csrc/f32_path.cu names:
    LayerNorm       transformer/ops.py:14-24                 eps 1e-5, biased variance
    Conv1D          transformer/ops.py:83-101                x . w + b, w [n_in, n_out]
    attention       factored_attention.py:82-108             q . k * dh^-1/2, softmax over the pattern's keys, . v
    keys            oracle.transformer_np.rows_attended      (factored_attention.py:123-228, 328-353); a previous-block
                                                             query in the first block attends a zero block: output 0
    block           transformer/transformer.py:62-86         x1 = x + c_proj(a); h = x1 + proj2(quick_gelu(fc(LN(x1))))

`layer_f64` takes every input row [n, L, width] (K / V are made of all of them, or of encoder_kv for attn_func 6) but
evaluates queries only at the positions asked for, so the dense layer at its last position costs one row of scores,
not an L x L matrix.

The bound (`bound="worst"` or `"stat"`) is carried through the layer as a vector of absolute errors per value: every
operation adds its own rounding error (local) and passes on the error of its inputs through the absolute value of its
derivative (first order): the worst-case model adds the input errors' absolute values through every product, the
statistical one their root sum of squares (the roundings of different outputs are independent).  Local errors of a dot product of K terms p_k with result y:
    worst  gamma_{K+r} (sum_k |p_k| + |bias| + |residual|)        (any summation order; r roundings after the sum)
    stat   3 u sqrt(K) (||p||_2 + |y|) + r u (|y| + |bias| + |residual|)
`worst` is the classical bound and holds for any order of the fp32 additions.  `stat` is its size in practice:
f32_path.cu sums every dot product in one fma chain, so each rounding errs by at most u times the partial sum it rounds.
The partial sums are about ||p||_2 sqrt(m / K) (random signs) plus y m / K (drift).  So the K roundings are independent
errors whose sum has a standard deviation below u sqrt(K) (||p||_2 + |y|) / sqrt(3), and 3 u sqrt(K) puts each output
five standard deviations away.  LayerNorm's sums use the reduction depth of layernorm_f32_kernel (256 threads: a serial
stretch of ceil(W / 256), five shuffle levels, eight warp partials), so both models share its worst-case term.
"""
import math

import numpy as np
import torch

from .transformer_np import rows_attended

U = 2.0 ** -24
C_STAT = 3.0


def gamma(k):
    return k * U / (1 - k * U)


def ln_depth(width):
    """the longest chain of fp32 additions in layernorm_f32_kernel's sums"""
    return -(-width // 256) + 5 + 8


def layer_norm(x, g, b, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    r = torch.rsqrt((d * d).mean(-1, keepdim=True) + eps)
    return d * r * g + b


def layer_norm_bound(x, ex, g, b, eps=1e-5):
    """LayerNorm rows x (error ex, or None) -> (y, bound on |fl(y) - y|) for layernorm_f32_kernel"""
    W = x.shape[-1]
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    r = torch.rsqrt((d * d).mean(-1, keepdim=True) + eps)
    y = d * r * g + b
    D = ln_depth(W)
    # mean: |mu^ - mu| <= gamma_D mean|x|; d: one subtraction; var: gamma_{D+2} relative; r: sqrt, divide, add eps
    loc = g.abs() * r * (gamma(D + 1) * x.abs().mean(-1, keepdim=True) + gamma(D + 8) * d.abs()) \
        + 3 * U * ((d * r * g).abs() + b.abs())
    if ex is None:
        return y, loc
    eb = ex.mean(-1, keepdim=True)
    ed = ex + eb
    prop = g.abs() * r * (ed + d.abs() * r * r * (d.abs() * ed).mean(-1, keepdim=True))
    return y, prop + loc


def _dot_loc(model, K, sum_abs, l2, y, r, extra):
    """local rounding error of a K-term fp32 dot product y (see the module docstring); extra = |bias| + |residual|"""
    if model == "worst":
        return gamma(K + r) * (sum_abs + extra)
    return C_STAT * U * math.sqrt(K) * (l2 + y.abs()) + r * U * (y.abs() + extra)


def _prop(model, e, w):
    """an input error e carried through the product e . w: worst case, or root-sum-square (independent errors)"""
    if model == "worst":
        return e @ w.abs()
    return torch.sqrt((e * e) @ (w * w))


def linear(x, ex, w, b, model=None, res=None, eres=None):
    """y = x . w + b (+ res) and, with a model, the bound on its fp32 error given the input errors ex / eres"""
    acc = x @ w
    y = acc + b if res is None else acc + b + res
    if model is None:
        return y, None
    K = x.shape[-1]
    extra = b.abs() if res is None else b.abs() + res.abs()
    loc = _dot_loc(model, K, x.abs() @ w.abs(), torch.sqrt((x * x) @ (w * w)), acc, 1 if res is None else 2, extra)
    e = loc if ex is None else loc + _prop(model, ex, w)
    if eres is not None:
        e = e + eres
    return y, e


def quick_gelu(z, ez=None):
    s = torch.sigmoid(1.702 * z)
    y = z * s
    if ez is None:
        return y, None
    # -1.702 z, expf (2 ulp), 1 +, 1 /, z * : |dy/dz| = |s + 1.702 z s (1 - s)|
    return y, (s + 1.702 * z * s * (1 - s)).abs() * ez + 8 * U * y.abs()


def attended_keys(attn_func, p, bc, prime, n_keys, shift=0):
    """key rows of the query at position p, or None for the zero block; `shift` moves the whole set (rows outside
    [0, n_keys) dropped) - the wrong pattern the sensitivity checks compare against"""
    if attn_func == 6:
        rows = np.arange(n_keys)
    elif attn_func == 3:
        blk = p // bc
        if blk == 0 and shift == 0:
            return None
        rows = np.arange((blk - 1) * bc, blk * bc)
    else:
        rows = rows_attended(attn_func, p, bc, prime)[1]
    rows = rows + shift
    rows = rows[(rows >= 0) & (rows < n_keys)]
    return rows if len(rows) else None


def layer_f64(p, x, queries, attn_func, n_head, block_ctx=None, prime=None, encoder_kv=None, shift=0, bound=None):
    """One layer in float64.

    p: {reference state-dict name relative to the block (`ln_0.weight`, `attn.c_attn.w`, ...): float64 tensor}
    x: [n, L, width] float64 input rows (positions 0 .. L-1); queries: positions to evaluate (< L)
    block_ctx: n_ctx // blocks; prime: the padded prime length (transformer_np.prime_len_padded); encoder_kv:
    [n, encoder_dims, width] for attn_func 6; shift: evaluate another key set (attended_keys); bound: None, "worst" or
    "stat" (module docstring).
    Returns {"y": [n, Q, width], "w": [n, heads, Q, keys] attention weights, "k", "v": [n, keys, n_state] (error
    bounds "ey", "ew", "ek", "ev" with a bound model)}."""
    n, L, W = x.shape
    qpos = torch.as_tensor(list(queries), dtype=torch.long, device=x.device)
    m = bound
    u0, eu0 = layer_norm_bound(x, None, p["ln_0.weight"], p["ln_0.bias"]) if m else \
        (layer_norm(x, p["ln_0.weight"], p["ln_0.bias"]), None)
    if attn_func == 6:
        S = p["attn.c_attn.w"].shape[1]
        uq, euq = u0[:, qpos], None if eu0 is None else eu0[:, qpos]
        q, eq = linear(uq, euq, p["attn.c_attn.w"], p["attn.c_attn.b"], m)
        kv, ekv = linear(encoder_kv, None, p["attn.c_enc_kv.w"], p["attn.c_enc_kv.b"], m)
        k, v = kv[..., :S], kv[..., S:]
        ek, ev = (None, None) if ekv is None else (ekv[..., :S], ekv[..., S:])
    else:
        S = p["attn.c_attn.w"].shape[1] // 3
        qkv, eqkv = linear(u0, eu0, p["attn.c_attn.w"], p["attn.c_attn.b"], m)
        q, k, v = qkv[:, qpos, :S], qkv[..., S:2 * S], qkv[..., 2 * S:]
        eq, ek, ev = (None, None, None) if eqkv is None else (eqkv[:, qpos, :S], eqkv[..., S:2 * S], eqkv[..., 2 * S:])
    H, Lk = n_head, k.shape[1]
    dh = S // H
    scale2 = (1.0 / math.sqrt(math.sqrt(dh))) ** 2
    Q = len(qpos)
    a = torch.zeros(n, Q, S, dtype=x.dtype, device=x.device)
    ea = torch.zeros_like(a) if m else None
    wts = torch.zeros(n, H, Q, Lk, dtype=x.dtype, device=x.device)
    ew = torch.zeros_like(wts) if m else None
    for i, pos in enumerate(queries):
        rows = attended_keys(attn_func, int(pos), block_ctx, prime, Lk if attn_func == 6 else L, shift)
        if rows is None:
            continue
        idx = torch.as_tensor(rows, device=x.device)
        qh = q[:, i].reshape(n, H, 1, dh)
        kh = k[:, idx].reshape(n, -1, H, dh).permute(0, 2, 3, 1)          # [n, H, dh, nk]
        vh = v[:, idx].reshape(n, -1, H, dh).permute(0, 2, 1, 3)          # [n, H, nk, dh]
        s = (qh @ kh) * scale2                                           # [n, H, 1, nk]
        pr = torch.softmax(s, -1)
        o = pr @ vh                                                      # [n, H, 1, dh]
        a[:, i] = o.reshape(n, S)
        wts[:, :, i, idx] = pr[:, :, 0]
        if not m:
            continue
        nk = len(rows)
        eqh = eq[:, i].reshape(n, H, 1, dh)
        ekh = ek[:, idx].reshape(n, -1, H, dh).permute(0, 2, 3, 1)
        evh = ev[:, idx].reshape(n, -1, H, dh).permute(0, 2, 1, 3)
        raw = qh @ kh
        es = scale2 * (_prop(m, ekh.transpose(-1, -2), qh.transpose(-1, -2)).transpose(-1, -2) + _prop(m, eqh, kh)
                       + _dot_loc(m, dh, qh.abs() @ kh.abs(), torch.sqrt((qh * qh) @ (kh * kh)), raw, 1, 0.0))
        # softmax: |d pr_j| <= pr_j (|ds_j| + sum_k pr_k |ds_k|); own rounding: s - max, expf (2 ulp), the row sum,
        # 1 / l and the product
        sum_loc = gamma(nk) if m == "worst" else C_STAT * U * math.sqrt(nk) * 2
        epr = pr * (es + (pr * es).sum(-1, keepdim=True)) + pr * (6 * U + sum_loc)
        ew[:, :, i, idx] = epr[:, :, 0]
        eo = _prop(m, epr, vh) + _prop(m, evh.transpose(-1, -2), pr.transpose(-1, -2)).transpose(-1, -2) \
            + _dot_loc(m, nk, pr @ vh.abs(), torch.sqrt((pr * pr) @ (vh * vh)), o, 0, 0.0)
        ea[:, i] = eo.reshape(n, S)
    xq = x[:, qpos]
    x1, ex1 = linear(a, ea, p["attn.c_proj.w"], p["attn.c_proj.b"], m, res=xq, eres=None)
    if m:
        v1, ev1 = layer_norm_bound(x1, ex1, p["ln_1.weight"], p["ln_1.bias"])
    else:
        v1, ev1 = layer_norm(x1, p["ln_1.weight"], p["ln_1.bias"]), None
    f, ef = linear(v1, ev1, p["mlp.c_fc.w"], p["mlp.c_fc.b"], m)
    g, eg = quick_gelu(f, ef)
    y, ey = linear(g, eg, p["mlp.c_proj.w"], p["mlp.c_proj.b"], m, res=x1, eres=ex1)
    out = {"y": y, "w": wts, "k": k, "v": v}
    if m:
        out.update(ey=ey, ek=ek, ev=ev, ew=ew)
    return out


def block_params(sd, d, device="cpu", fp16_params=False):
    """float64 tensors of layer d from a reference state dict {`_attn_mods.{d}.<name>`: array}; with fp16_params the
    Conv1D weights are first rounded to fp16, as make_models.py stores them"""
    pre = f"_attn_mods.{d}."
    out = {}
    for k, v in sd.items():
        if k.startswith(pre):
            a = np.asarray(v, np.float32)
            if fp16_params and k.endswith(".w"):
                a = a.astype(np.float16).astype(np.float32)
            out[k[len(pre):]] = torch.from_numpy(a).to(device=device, dtype=torch.float64)
    return out


def stack_f64(sd, x, attn_funcs, n_head, block_ctx=None, prime=None, encoder_kv=None, fp16_params=False, queries=None):
    """every layer of a stack in float64, in forward mode: x [n, L, width] -> [n, L, width] (all positions), or the rows
    of `queries` of the last layer (earlier layers still run over every row: later layers attend them)"""
    h = x
    for d, af in enumerate(attn_funcs):
        last = d == len(attn_funcs) - 1
        qs = queries if (last and queries is not None) else range(h.shape[1])
        h = layer_f64(block_params(sd, d, x.device, fp16_params), h, qs, af, n_head, block_ctx, prime, encoder_kv)["y"]
    return h
