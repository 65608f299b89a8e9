"""The decode step's attention (csrc/decode_engine.cu attn_geom / attn_tile_rows / attn_nsplit / attn_item / attn_prefetch),
restated for tests, with a float64 attention of one query and a first-order bound on the kernel's error against it.

TEST INFRASTRUCTURE ONLY (only tests/ may import it).  numpy.

Layout (restated exactly):
    attn_geom       per pattern: rows attended R, first cache row `base`, whether the current token is the last attended
                    row (`cur`), and the cache row the current token's k / v is written to (`wrow`, -1: none)
    cache rows      dense and prime: row p; block: ring of bc rows (p % bc); transpose: (p % bc) * blocks + p / bc;
                    prev: a two-block ring ((p / bc) & 1) * bc + p % bc, read at ((p / bc + 1) & 1) * bc; encoder: row r
    split           ns = 1 + [ncache > RC-1] + [ncache > 2(RC-1)] + [ncache > 3(RC-1)], at most gmax = G / (B H), at least 1
    parts           part s holds cached rows [ncache s / ns, ncache (s+1) / ns) (div_small); the last part also holds the
                    current token, appended to its last tile
    tiles           trows = RC - 1 cached rows per tile, ntiles = max(1, ceil((i1 - i0) / trows))
    items           item it = (b H + h) ns + s runs on CTA it % G (it = c, c + G, ...); only a CTA's first item (it < G)
                    finds its first tile prefetched, and only if R > 0

Attention (float64, the kernel's reference rounding points kept):  s_j = fp16(fp32(fp16(q . k_j) * scale2)) with
scale2 = float(dh^-1/2) (engine.cuh attn_scale2), p = softmax(s) and a = sum_j p_j v_j in float64.

Bound on |a_kernel - a64| per output dim (`bound`), the sum of:
  (a) score rounding: the fp32 tensor-core q . k_j is within e_j = gamma(dhp + 2) sum_d |q_d k_jd| of the exact product
      (every addition of an m16n8k16 MMA and the c0 + c1 add err by at most 2^-23 relative, truncation; 17 terms per
      MMA over dhp / 32 MMAs per chain is at most dhp + 2 additions); the roundings after it are monotone, so
      s_kernel,j lies in [f(qk - e_j), f(qk + e_j)] and |ds_j| <= the larger distance to s_j.  Weights then move by
      factors within e^{+-ds_j}, which moves the normalised average by at most
      sum_j p_j |v_j - a| (e^{ds_j} - 1) / (1 - sum_j p_j (1 - e^{-ds_j})).
  (b) P rounding: P is rounded to fp16 unnormalised, relative to its tile's running maximum m_t within its part; the
      row sum l does not see that rounding, so each key costs (2^-11 p_j + 2^-25 e^{m_t - M} / L) |v_j|: half an fp16 ulp
      relative for a normal P, half the subnormal spacing 2^-24 absolute for a subnormal one (M the global maximum,
      L = sum_j e^{s_j - M}).
  (c) P.V, rescales and merge: the fp32 P.V MMAs (17 terms per MMA, at most 4 MMAs per tile), one multiply and one add
      per `corr` rescale of a running output, one per merge weight, the final reciprocal or division, and the expf of
      P, corr and the merge weights (2 ulps each, the CUDA guide's bound) make a chain of n operations of relative
      error 2^-23 each: gamma(n) sum_j p_j |v_j|.
  (d) the row sum l: the unrounded fp32 p summed by a 64-lane tree (6 additions), rescaled and added once per tile,
      merged once per part, with the same expf errors: gamma(n_l) |a|.
  (e) output rounding: half an fp16 ulp of |a| + (a) + (b) + (c) + (d) (2^-25 at least: the subnormal spacing).
Cross terms between (a) .. (d) are second order (below 2^-40 relative) and are not charged."""
import math

import numpy as np

from oracle.transformer_np import rows_attended

U32 = 2.0 ** -23


def attn_tile_rows(dhp):
    r = (12288 // dhp) & ~15
    return 16 if r < 16 else (64 if r > 64 else r)


def head_dim_pad(dh):
    return (dh + 15) // 16 * 16


def attn_scale2(dh):
    sc = 1.0 / math.sqrt(math.sqrt(dh))
    return np.float32(sc * sc)


def div_small(x, d):
    if d == 1:
        return x
    if d == 2:
        return x >> 1
    if d == 4:
        return x >> 2
    return (x * 43691) >> 17


def prime_pad_len(prime_len, blocks):
    return (prime_len // blocks + 1) * blocks if blocks > 0 else 0


class Geom:
    """the attention geometry of one engine: heads, head dim, context, blocks, prime, encoder rows, tile rows RC, SMs G"""

    def __init__(self, *, heads, dh, n_ctx, blocks, prime_len=0, enc_dims=0, G=132, RC=None):
        self.H, self.dh, self.dhp = heads, dh, head_dim_pad(dh)
        self.n_ctx, self.blocks = n_ctx, blocks
        self.bc = n_ctx // blocks if blocks > 0 else n_ctx
        self.prime_pad = prime_pad_len(prime_len, blocks)
        self.enc_dims, self.G = enc_dims, G
        self.RC = attn_tile_rows(self.dhp) if RC is None else RC
        self.trows = self.RC - 1
        self.swizzled = (self.dhp // 8) % 8 == 0
        self.scale2 = attn_scale2(dh)

    def rows_of(self, af):
        """cache rows per (sample, head) of a layer (engine.cuh cache_rows_for)"""
        return {0: self.n_ctx, 1: self.bc, 2: self.n_ctx, 3: 2 * self.bc, 6: self.enc_dims, 7: self.prime_pad}[af]


def attn_geom(g, af, p, mutate=None):
    """(R, base, cur, wrow) of the query at position p (csrc/decode_engine.cu attn_geom).  mutate names a deliberately
    wrong layout, for tests that show the checks catch it: "base+1", "transpose_as_p", "prev_swap"."""
    bc, pm, pd = g.bc, p % g.bc, p // g.bc
    if af == 0:
        R, base, cur, wrow = p + 1, 0, 1, p
    elif af == 1:
        R, base, cur, wrow = pm + 1, 0, 1, pm
    elif af == 2:
        base = pm * g.blocks
        R, cur, wrow = pd + 1, 1, (p if mutate == "transpose_as_p" else base + pd)
    elif af == 3:
        R = bc if p >= bc else 0
        base = (pd & 1) * bc if mutate == "prev_swap" else ((pd + 1) & 1) * bc
        cur, wrow = 0, (pd & 1) * bc + pm
    elif af == 7:
        R, base = min(p + 1, g.prime_pad), 0
        cur = 1 if p < g.prime_pad else 0
        wrow = p if p < g.prime_pad else -1
    elif af == 6:
        R, base, cur, wrow = g.enc_dims, 0, 0, -1
    else:
        raise ValueError(af)
    if mutate == "base+1":
        base += 1
    return R, base, cur, wrow


def ncache_of(R, cur):
    return R - (1 if (R > 0 and cur) else 0)


def attn_nsplit(g, gmax, ncache):
    cap = g.RC - 1
    ns = 1 + (ncache > cap) + (ncache > 2 * cap) + (ncache > 3 * cap)
    return max(1, min(ns, gmax))


def gmax_of(g, B):
    return max(1, g.G // (B * g.H))


def partition(g, ncache, ns, cur):
    """the parts of one (sample, head): [dict(s, i0, i1, tiles=[(r0, nr cached, holds the current token)])]"""
    out = []
    for s in range(ns):
        i0, i1 = div_small(ncache * s, ns), div_small(ncache * (s + 1), ns)
        nt = max(1, (i1 - i0 + g.trows - 1) // g.trows)
        tiles = []
        for ti in range(nt):
            r0 = i0 + ti * g.trows
            nr = max(0, min(g.trows, i1 - r0))
            tiles.append((r0, nr, bool(cur and s == ns - 1 and ti == nt - 1)))
        out.append(dict(s=s, i0=i0, i1=i1, tiles=tiles))
    return out


def items(g, B, ns, R):
    """the attention items of one launch: dict(it, b, h, s, cta, prefetched) (the loop `it = c; it += G` and attn_prefetch)"""
    out = []
    for it in range(B * g.H * ns):
        bh = div_small(it, ns)
        s, b = it - bh * ns, bh // g.H
        out.append(dict(it=it, b=b, h=bh - b * g.H, s=s, cta=it % g.G, prefetched=bool(it < g.G and R > 0)))
    return out


class CacheRows:
    """which position's k / v each cache row of one pattern holds, as the kernel writes them step by step; read(p)
    gives the attended positions of the query at p in the kernel's order (cached rows, then the current token)"""

    def __init__(self, g, af, mutate=None):
        self.g, self.af, self.mutate = g, af, mutate
        self.reset()

    def reset(self):
        rows = self.g.rows_of(self.af) + 2               # + 2: room for the off-by-one mutation to read past the end
        self.row = np.full(rows, -1, np.int64)
        if self.af == 6:
            self.row[:self.g.enc_dims] = np.arange(self.g.enc_dims)

    def read(self, p):
        R, base, cur, wrow = attn_geom(self.g, self.af, p, self.mutate)
        if R == 0:
            return "zeros", np.zeros(0, np.int64), 0
        nc = ncache_of(R, cur)
        pos = self.row[base:base + nc].copy()
        return "rows", np.concatenate([pos, [p]]) if cur else pos, cur

    def write(self, p):
        wrow = attn_geom(self.g, self.af, p, self.mutate)[3]
        if wrow >= 0:
            self.row[wrow] = p


def expected_rows(g, af, p):
    """rows_attended (the reference's pattern) for the same query, or encoder rows 0 .. enc_dims - 1"""
    if af == 6:
        return "rows", np.arange(g.enc_dims)
    return rows_attended(af, p, g.bc, g.prime_pad)


# ---- scores and the float64 attention ------------------------------------------------------------------------------
def f16(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float16)


def score_of(qk, scale2):
    """fp16(fp32(fp16(qk) * scale2)) of float64 q.k values (the fp32 accumulator rounded, then as attn_scores)"""
    return (f16(qk).astype(np.float32) * np.float32(scale2)).astype(np.float16).astype(np.float64)


def qk_error(q, K, dhp):
    """e_j: the tensor cores' accumulation bound on q . k_j (term (a)); plus a float64 margin for the exact product"""
    n = dhp + 2
    gam = n * U32 / (1 - n * U32)
    mag = np.abs(K.astype(np.float64)) @ np.abs(q.astype(np.float64))
    return gam * mag + 2.0 ** -50 * mag


def attend64(q, K, V, scale2):
    """one query against rows K, V (fp16 values, [n, dh]): (s, p, a) in float64 with the kernel's score roundings"""
    qk = K.astype(np.float64) @ q.astype(np.float64)
    s = score_of(qk, scale2)
    w = np.exp(s - s.max())
    p = w / w.sum()
    return s, p, p @ V.astype(np.float64)


def bound(q, K, V, g, parts):
    """the per-dim bound on |a_kernel - a64| (module docstring) of one query whose rows K, V are in the kernel's order
    and split as `parts` (partition())"""
    dhp = g.dhp
    qk = K.astype(np.float64) @ q.astype(np.float64)
    s, p, a = attend64(q, K, V, g.scale2)
    e = qk_error(q, K, dhp)
    ds = np.maximum(np.abs(score_of(qk - e, g.scale2) - s), np.abs(score_of(qk + e, g.scale2) - s))
    V64 = V.astype(np.float64)
    up, dn = np.expm1(ds), -np.expm1(-ds)
    term_a = (p * up) @ np.abs(V64 - a) / (1 - float(p @ dn))
    # (b): the running maximum of each key's tile, in its part (scores at their upper end f(qk + e))
    s_hi = score_of(qk + e, g.scale2)
    mt = np.empty_like(s)
    ntiles = 1
    for part in parts:
        m = -np.inf
        ntiles = max(ntiles, len(part["tiles"]))
        for r0, nr, withcur in part["tiles"]:
            idx = list(range(r0, r0 + nr)) + ([len(s) - 1] if withcur else [])
            if idx:
                m = max(m, s_hi[idx].max())
                mt[idx] = m
    M = s.max()
    L = np.exp(s - M).sum()
    term_b = (2.0 ** -11 * p + 2.0 ** -25 * np.exp(mt - M) / L) @ np.abs(V64)
    ns = len(parts)
    n_c = 17 * 4 + 2 * ntiles + 2 * ns + 2 + 2 * (ntiles + 1 + ns)
    term_c = n_c * U32 / (1 - n_c * U32) * (p @ np.abs(V64))
    n_l = 6 + 2 * ntiles + 2 * ns + 2 + 2 * (ntiles + 1 + ns)
    term_d = n_l * U32 / (1 - n_l * U32) * np.abs(a)
    tot = term_a + term_b + term_c + term_d
    mag = np.abs(a) + tot
    ulp = np.maximum(2.0 ** (np.floor(np.log2(np.maximum(mag, 2.0 ** -14))) - 10), 2.0 ** -24)
    return tot + 0.5 * ulp, a, dict(a=term_a, b=term_b, c=term_c, d=term_d)


# ---- a numpy emulation of the kernel's arithmetic (for the bound's own tests) --------------------------------------
def emulate(q, K, V, g, parts, qk_shift=None, mutate=None):
    """attn_item's arithmetic for one query: fp16 scores from an fp32 q.k (moved by qk_shift, in [-1, 1] units of the
    bound e_j, to stand for the tensor cores' accumulation), flash-style fp32 softmax per tile with the running maximum
    of its part, fp16 unnormalised P, fp32 P.V per tile, the corr rescale, then the fixed merge in part order and the
    fp16 output.  mutate: "no_corr" (the running output is not rescaled), "merge_no_w" (the merge drops
    expf(m_q - M)), "cur_wrong_tile" (the current token's k / v land in the other tile region, so the last tile's appended
    row holds stale data, here zeros)."""
    f32 = np.float32
    qk = K.astype(np.float64) @ q.astype(np.float64)
    if qk_shift is not None:
        qk = qk + qk_shift * qk_error(q, K, g.dhp)
    s_all = (f16(qk).astype(f32) * f32(g.scale2)).astype(np.float16).astype(f32)
    V32 = V.astype(np.float16).astype(f32)
    res = []
    for part in parts:
        m_run, l_run, o = f32(-np.inf), f32(0), np.zeros(V.shape[1], f32)
        tiles = part["tiles"]
        for ti, (r0, nr, withcur) in enumerate(tiles):
            idx = list(range(r0, r0 + nr))
            sv, vv = s_all[idx], V32[idx]
            if withcur:
                if mutate == "cur_wrong_tile":
                    cs, cv = f32(score_of(0.0, g.scale2)), np.zeros(V.shape[1], f32)
                else:
                    cs, cv = s_all[-1], V32[-1]
                sv, vv = np.append(sv, cs), np.vstack([vv, cv[None]])
            m_new = f32(max(m_run, sv.max())) if len(sv) else m_run
            corr = f32(np.exp(f32(m_run - m_new))) if np.isfinite(m_run) else f32(0)
            pt = np.exp((sv - m_new).astype(f32)).astype(f32)
            l_run = f32(f32(l_run * corr) + f32(pt.sum(dtype=f32)))
            m_run = m_new
            P = pt.astype(np.float16).astype(f32)
            ot = (P.astype(np.float64) @ vv.astype(np.float64)).astype(f32)
            if ti > 0:
                ot = (ot + (o if mutate == "no_corr" else (o * corr).astype(f32))).astype(f32)
            o = ot
        res.append((m_run, l_run, o))
    if len(res) == 1:
        m_run, l_run, o = res[0]
        inv = f32(f32(1) / l_run)
        return (o * inv).astype(f32).astype(np.float16)
    M = f32(max(r[0] for r in res))
    Ls, out = f32(0), np.zeros(V.shape[1], f32)
    for m_q, l_q, o_q in res:
        w = f32(1) if mutate == "merge_no_w" else f32(np.exp(f32(m_q - M)))
        Ls = f32(Ls + f32(l_q * w))
        out = (out + (o_q * w).astype(f32)).astype(f32)
    return (out / Ls).astype(f32).astype(np.float16)
