"""The decode engine's LayerNorm, restated exactly: its fixed-point row statistics and its fp16 staging.

TEST INFRASTRUCTURE ONLY (only tests/ may import it).  numpy; int64 for the statistics words, float32 / float64 with the
roundings csrc/decode_engine.cu performs, so that the GPU tests can demand bit equality with the kernel.

What is restated (csrc/decode_engine.cu):
    fx_sum(x)       __float2ll_rn(x * 65536.0f)                              fp32 product, round to nearest even
    fx_sq(x)        __float2ll_rn(fminf(x * x, 16777216.0f) * 16384.0f)
    words           [63:52] contributing CTAs, [51:0] value; the sum word carries kSumBias = 2^41 per contribution
    row_statistics  rk = double(1.0f / K); m = val * 2^-16 * rk; var = max(fma(rk, sq * 2^-14, -fl(m * m)), 0)
                    (an explicit fma: one rounding of E[x^2] - m^2)
                    rstd = 1.0f / sqrtf(float(var) + 1e-5f); nmr = -float(m) * rstd
    staging         fp16(fmaf(fmaf(x, rstd, nmr), gamma, beta))

The statistics are a property of the row alone: every value is rounded per element to its grid before the integer
sums, so neither the order of the CTAs nor the split of the row into column slices can change them.  That is why the
kernel can be held to them bit for bit."""
from fractions import Fraction

import numpy as np

CNT_SHIFT = 52
VAL_MASK = (1 << CNT_SHIFT) - 1
SUM_BIAS = 1 << 41
SQ_CLAMP = np.float32(2.0 ** 24)


def _rn_ll(v):
    """__float2ll_rn of float32 values (round half to even; every fp32 value used here is far inside int64)"""
    return np.rint(v.astype(np.float64)).astype(np.int64)


def fx_sum(x):
    x = np.asarray(x, np.float32)
    return _rn_ll(x * np.float32(65536.0))


def fx_sq(x):
    x = np.asarray(x, np.float32)
    return _rn_ll(np.minimum(x * x, SQ_CLAMP) * np.float32(16384.0))


def stat_words(x, G):
    """the two statistics words of every row of x [..., K] (fp16 values) after all G CTAs have contributed (the CTAs
    without columns add the bias and the count only): (sum word, sum-of-squares word) as uint64"""
    s = fx_sum(x).sum(-1) + G * SUM_BIAS
    q = fx_sq(x).sum(-1)
    cnt = np.uint64(G) << np.uint64(CNT_SHIFT)
    return cnt + s.astype(np.uint64), cnt + q.astype(np.uint64)


def row_statistics(x, G=1):
    """(mean, var, rstd, nmr) of every row of x [..., K] as the kernel derives them from its words: mean and var in
    float64 (what the format delivers), rstd and nmr in float32 (what the staging multiplies with)"""
    x = np.asarray(x, np.float32)
    K = x.shape[-1]
    ws, wq = stat_words(x, G)
    val = (ws & np.uint64(VAL_MASK)).astype(np.int64) - G * SUM_BIAS
    sq = (wq & np.uint64(VAL_MASK)).astype(np.int64)
    rk = np.float64(np.float32(1.0) / np.float32(K))
    m = val.astype(np.float64) * (1.0 / 65536.0) * rk
    # the kernel's explicit fma(rk, sq * 2^-14, -(m * m)): the product with rk is not rounded on its own
    var = dfma(np.full_like(m, rk), sq.astype(np.float64) * (1.0 / 16384.0), -(m * m))
    var = np.maximum(var, 0.0)
    rstd = np.float32(1.0) / np.sqrt(var.astype(np.float32) + np.float32(1e-5))
    nmr = -m.astype(np.float32) * rstd
    return m, var, rstd.astype(np.float32), nmr.astype(np.float32)


def dfma(a, b, c):
    """fma in float64, element by element: a * b + c exact (Python fractions), then one rounding"""
    a, b, c = (np.asarray(v, np.float64) for v in np.broadcast_arrays(a, b, c))
    out = np.empty(a.shape, np.float64)
    for i in np.ndindex(a.shape):
        out[i] = float(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
    return out


def fmaf(a, b, c):
    """fmaf in numpy: a * b + c rounded once to float32.  The float64 product of two floats is exact; the float64 sum
    is rounded, and its error e is recovered exactly (two-sum), so the one case where rounding the float64 sum to
    float32 would round twice - the sum lands exactly on a float32 midpoint - is decided by the sign of e."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    other = 2.0 * s - r64                       # the float32 on the other side of s when s is a midpoint
    mid = (other != r64) & (other.astype(np.float32).astype(np.float64) == other)
    toward_other = mid & (e != 0) & (np.sign(e) == np.sign(other - r64))
    return np.where(toward_other, other.astype(np.float32), r).astype(np.float32)


def staged(x, gamma, beta, G=1):
    """the fp16 LayerNorm rows the kernel stages: fp16(fmaf(fmaf(x, rstd, nmr), gamma, beta)), x [..., K] fp16 values"""
    x = np.asarray(x, np.float32)
    _, _, rstd, nmr = row_statistics(x, G)
    t = fmaf(x, rstd[..., None], nmr[..., None])
    return fmaf(t, np.asarray(gamma, np.float32), np.asarray(beta, np.float32)).astype(np.float16)


def quick_gelu16(y):
    """the kernel's quick_gelu of fp16 values y (three fp16 roundings, csrc/decode_engine.cu quick_gelu_f), and for every
    element whether its float32 pre-rounding value lies within 2 float32 ulps of an fp16 rounding boundary (numpy's
    expf and the device's may differ there by the 2 ulps the CUDA guide allows)"""
    x = np.asarray(y, np.float32)
    z = (np.float32(1.702) * x).astype(np.float16).astype(np.float32)
    d = np.float32(1.0) + np.exp(-z)
    s32 = np.float32(1.0) / d
    s = s32.astype(np.float16).astype(np.float32)
    out32 = x * s
    near = _near_f16_boundary(s32) | _near_f16_boundary(out32)
    return out32.astype(np.float16), near


def _near_f16_boundary(v, ulps=2):
    v = np.asarray(v, np.float32)
    lo, hi = v, v
    for _ in range(ulps):
        lo = np.nextafter(lo, np.float32(-np.inf))
        hi = np.nextafter(hi, np.float32(np.inf))
    return lo.astype(np.float16) != hi.astype(np.float16)
