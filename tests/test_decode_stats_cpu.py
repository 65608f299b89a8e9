"""The decode engine's LayerNorm statistics format (oracle/decode_stats.py restates csrc/decode_engine.cu), on the CPU.

  * the value field of a statistics word never reaches the count bits, for every CTA's contribution and every sum of
    them, at the columns each CTA owns in the plans of the baseline configurations and at K = 8192, with rows of
    +-65504 (the fp16 maximum);
  * an analytic worst-case bound on the variance the words deliver, held on rows built to push every rounding the
    same way;
  * the format's envelope: the staged LayerNorm output against the exact float64 LayerNorm of the same fp16 row, in
    fp16 ulps, by row std, by |mean| / std, for constant rows and past the 4096 clamp of the squares (the table in
    DESIGN.md "Numerics" is this test's output).
The GPU half (tests/test_gpu_decode_geometry.py) holds the kernel to the restatement bit for bit."""
from fractions import Fraction

import numpy as np
import pytest

from oracle.decode_stats import (CNT_SHIFT, SUM_BIAS, fmaf, fx_sq, fx_sum, row_statistics, staged)
from test_decode_plan_cpu import CONFIGS, plan

F16_MAX = 65504.0


def contributions(x, owned):
    """the values one LayerNorm's CTAs add to a row's two words: owned = [CTA] -> its columns"""
    s = np.array([SUM_BIAS + int(fx_sum(x[c]).sum()) for c in owned], dtype=object)
    q = np.array([int(fx_sq(x[c]).sum()) for c in owned], dtype=object)
    return s, q


def owned_columns(name):
    """the residual-stream columns each CTA of the 132-SM plan finishes (proj / proj2 columns, statistics producers)"""
    _, info, cols = plan(name)
    ks = info.k_split
    out = []
    for u in range(info.units):
        g0, ncg = int(cols[u, 0, 1, 0]), int(cols[u, 0, 1, 1])
        pairs = ncg * 4 // ks
        for r in range(ks):
            c0 = g0 * 8 + 2 * r * pairs
            out.append(np.arange(c0, c0 + 2 * pairs))
    return out


def assert_fields_hold(x, owned):
    s, q = contributions(x, owned)
    lim = 1 << CNT_SHIFT
    for v in (s, q):
        assert all(0 <= int(c) < lim for c in v)            # every red alone
        assert 0 <= int(v.sum()) < lim                        # and every partial sum: contributions are >= 0
    return int(s.sum()), int(q.sum())


@pytest.mark.parametrize("name", [n for n in CONFIGS if n != "tiny"])
def test_value_field_never_reaches_count_bits(name):
    owned = owned_columns(name)
    G = len(owned)
    assert G == 132 and len(owned) < (1 << (64 - CNT_SHIFT))
    W = CONFIGS[name][0]
    assert sorted(np.concatenate(owned).tolist()) == list(range(W))
    for row in (np.full(W, F16_MAX), np.full(W, -F16_MAX), F16_MAX * (1 - 2 * (np.arange(W) % 2))):
        assert_fields_hold(row.astype(np.float32), owned)


def test_value_field_holds_at_8192_columns():
    """K = 8192 (the largest width the format was sized for), 64 columns per CTA (the most any plan gives one CTA: 8
    column groups at K split 1) and 132 CTAs, the rest empty contributors"""
    K, G = 8192, 132
    owned = [np.arange(i, min(i + 64, K)) for i in range(0, K, 64)]
    owned += [np.arange(0)] * (G - len(owned))
    for row in (np.full(K, F16_MAX), np.full(K, -F16_MAX)):
        s, q = assert_fields_hold(row.astype(np.float32), owned)
    assert s < (1 << CNT_SHIFT) and q < (1 << CNT_SHIFT)
    # the margin left: the sum field's highest value against 2^52
    print(f"K 8192 at +65504: sum field {s / 2 ** 52:.3f} of 2^52, squares field {q / 2 ** 52:.3f}")


def exact_mean_var(x):
    """mean and (biased) variance of an fp16 row, exactly: every fp16 value is an integer multiple of 2^-24, so the sums
    are integers and the variance is one fraction, rounded once to float64"""
    X = [int(v) for v in (np.asarray(x, np.float16).astype(np.float64) * 2.0 ** 24)]
    K = len(X)
    s1, s2 = sum(X), sum(v * v for v in X)
    return float(Fraction(s1, K * 2 ** 24)), float(Fraction(K * s2 - s1 * s1, K * K * 2 ** 48))


def var_error_bound(x):
    """worst case of |var_words - var(x)| for an fp16 row x [K] with no |x| > 4096 (no clamp): fx_sum rounds each element
    by <= 2^-17, fx_sq by <= 2^-15; rk = fp32(1/K) errs by d <= 2^-24 relative; the float64 product for m and m * m
    each round by 2^-53 relative, the DFMA once more"""
    x = x.astype(np.float64)
    K = x.size
    rk = float(np.float32(1.0) / np.float32(K))
    d = abs(rk * K - 1.0)
    m, e2 = abs(x.mean()), (x * x).mean()
    u = 2.0 ** -53
    dm = (2.0 ** -17) * (1 + d) + (d + u) * (m + 2.0 ** -17)           # |m_words - mean|
    return (2.0 ** -15) * (1 + d) + d * e2 + 2 * m * dm + dm * dm + 3 * u * (m * m + e2)


def adversarial_rows(K, rng):
    f16 = np.arange(0, 0x7800, dtype=np.uint16).view(np.float16).astype(np.float64)    # the positive fp16 values < 32768
    f16 = f16[np.isfinite(f16) & (f16 <= 4096)]
    frac_s = (f16 * 65536) % 1.0
    frac_q = (f16 * f16 * 16384) % 1.0
    rows = []
    # every element's sum rounds down by almost half a grid step
    down_s = f16[(frac_s > 0.45) & (frac_s < 0.5)]
    # every element's square rounds down (or up) by almost half a step
    down_q = f16[(frac_q > 0.45) & (frac_q < 0.5)]
    up_q = f16[(frac_q > 0.5) & (frac_q < 0.55)]
    for pool in (down_s, down_q, up_q):
        for lo, hi in ((0, 2.0 ** -8), (2.0 ** -8, 1.0), (1.0, 64.0), (64.0, 4096.0)):
            p = pool[(pool > lo) & (pool <= hi)]
            if len(p):
                rows.append(rng.choice(p, K))
                rows.append(rng.choice(p, K) * rng.choice([-1.0, 1.0], K))
    # large |mean| / std: the 1 / K rounding against E[x^2]
    for mean in (1000.0, -250.0, 3000.0):
        rows.append((mean + rng.standard_normal(K)).astype(np.float16).astype(np.float64))
    return [r.astype(np.float16).astype(np.float32) for r in rows]


@pytest.mark.parametrize("K", [1104, 1920, 2048, 4800])
def test_variance_error_within_analytic_bound(K):
    rng = np.random.RandomState(K)
    worst = 0.0
    for x in adversarial_rows(K, rng):
        _, var, _, _ = row_statistics(x[None])
        exact = exact_mean_var(x)[1]
        ratio = abs(var[0] - exact) / var_error_bound(x)
        worst = max(worst, ratio)
        assert ratio <= 1.0, (K, float(x.mean()), float(x.std()), var[0], exact)
    print(f"K {K}: worst |var error| / analytic bound {worst:.3f}")
    assert worst > 0.1            # the rows do push the roundings: the bound is not vacuous here


def test_fmaf_rounds_once():
    """fmaf against exact rational arithmetic, on products that land on float32 midpoints"""
    rng = np.random.RandomState(0)
    a = rng.standard_normal(20000).astype(np.float32)
    b = rng.standard_normal(20000).astype(np.float32)
    # c = -(a * b) rounded to float32, nudged: the exact sum is the small rounding residue, often a midpoint case
    c = -(a.astype(np.float64) * b).astype(np.float32) + np.float32(2.0 ** -30) * rng.choice([-1, 0, 1], 20000)
    c = c.astype(np.float32)
    got = fmaf(a, b, c)
    for i in range(0, 20000, 7):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        assert got[i] == np.float32(float(exact)) or abs(Fraction(float(got[i])) - exact) <= \
            abs(Fraction(float(np.float32(float(exact)))) - exact)
    # an exact float32 midpoint (no low part) rounds to even
    one = np.float32(1.0)
    assert fmaf(one + np.float32(2.0 ** -23), one, np.float32(-(2.0 ** -24)))[()] == one


def ulps16(got, exact):
    """|got - exact| in fp16 ulps of exact (subnormal spacing below 2^-14)"""
    e = np.abs(exact)
    ulp = np.where(e < 2.0 ** -14, 2.0 ** -24, 2.0 ** (np.floor(np.log2(np.maximum(e, 2.0 ** -14))) - 10))
    return np.abs(got.astype(np.float64) - exact) / ulp


def envelope_row(x):
    """fp16 ulps of the staged LayerNorm (gamma 1, beta 0) against the exact float64 LayerNorm of the same fp16 row:
    the largest and the median in ulps of each exact value, and the largest absolute error in ulps of 1 (2^-10, the
    scale of a normalised row: near-zero outputs carry the absolute error of x * rstd + nmr, many of their own ulps)"""
    h = x.astype(np.float16)
    K = h.size
    y = staged(h[None], np.ones(K, np.float32), np.zeros(K, np.float32))[0]
    hd = h.astype(np.float64)
    mean, var = exact_mean_var(h)
    ex = (hd - mean) / np.sqrt(var + 1e-5)
    u = ulps16(y, ex)
    return float(u.max()), float(np.median(u)), float(np.abs(y.astype(np.float64) - ex).max() / 2.0 ** -10)


ENVELOPE_K = 2048
# DESIGN.md's envelope table: (row, |mean| / std) -> (max ulps, median ulps, max abs error / 2^-10).  A change of the
# statistics format or of the staging arithmetic moves these numbers.
ENVELOPE = {
    ('std 2^-10', '0'): (508.9, 67.86, 56.16),
    ('std 2^-10', '1'): (101.7, 66.09, 51.74),
    ('std 2^-10', '16'): (10.61, 7.123, 4.951),
    ('std 2^-10', '256'): (92.07, 57.98, 56.24),
    ('std 2^-8', '0'): (210.8, 145.7, 303),
    ('std 2^-8', '1'): (167.4, 114.2, 220.1),
    ('std 2^-8', '16'): (19.06, 13.08, 24.01),
    ('std 2^-8', '256'): (213.7, 155.1, 358.5),
    ('std 2^-6', '0'): (51.75, 5.712, 12.34),
    ('std 2^-6', '1'): (13.05, 1.11, 3.272),
    ('std 2^-6', '16'): (4.6, 2.938, 7.288),
    ('std 2^-6', '256'): (12.27, 8.895, 23.58),
    ('std 2^-4', '0'): (5.55, 0.2567, 1.22),
    ('std 2^-4', '1'): (0.879, 0.2532, 1.107),
    ('std 2^-4', '16'): (0.9361, 0.3448, 1.629),
    ('std 2^-4', '256'): (1.363, 0.2663, 0.9881),
    ('std 2^-2', '0'): (0.5169, 0.245, 1.012),
    ('std 2^-2', '1'): (0.5096, 0.254, 0.9992),
    ('std 2^-2', '16'): (0.551, 0.2855, 1.055),
    ('std 2^-2', '256'): (0.4986, 0.3196, 0.9934),
    ('std 2^0', '0'): (0.4998, 0.2439, 1.138),
    ('std 2^0', '1'): (0.5011, 0.2333, 0.9988),
    ('std 2^0', '16'): (0.4974, 0.1884, 0.9875),
    ('std 2^0', '256'): (0.476, 0.2752, 0.952),
    ('std 2^2', '0'): (0.4998, 0.2469, 0.9995),
    ('std 2^2', '1'): (0.5071, 0.2579, 0.9898),
    ('std 2^2', '16'): (0.8267, 0.2647, 0.9868),
    ('std 2^2', '256'): (1.57, 0.3287, 0.9627),
    ('std 2^4', '0'): (0.4999, 0.2491, 0.9683),
    ('std 2^4', '1'): (0.4996, 0.2615, 0.9987),
    ('std 2^4', '16'): (11.7, 0.2411, 0.9713),
    ('std 2^4', '256'): (1.013e+07, 6.847e+06, 1.966e+07),
    ('std 2^6', '0'): (0.4996, 0.2569, 0.9976),
    ('std 2^6', '1'): (0.4999, 0.2469, 0.9833),
    ('std 2^6', '16'): (1.036, 0.2408, 0.992),
    ('std 2^6', '256'): (np.inf, 2.571e+07, np.inf),
    ('std 2^8', '0'): (0.4994, 0.2575, 0.9677),
    ('std 2^8', '1'): (0.5036, 0.2462, 0.9895),
    ('std 2^8', '16'): (np.inf, 1.463e+08, np.inf),
    ('std 2^10', '0'): (0.5, 0.2457, 0.998),
    ('std 2^10', '1'): (4.161, 2.299, 6.195),
    ('std 2^10', '16'): (np.inf, np.inf, np.inf),
    ('constant 0.1', '-'): (1, 1, 6.104e-05),
    ('constant 7.0', '-'): (0, 0, 0),
    ('constant 1000.0', '-'): (3.277e+04, 3.277e+04, 2),
    ('std 1000, 0% of |x| > 4096', '0'): (0.5, 0.2468, 0.9775),
    ('std 3000, 18% of |x| > 4096', '0'): (355.4, 250.2, 713.6),
    ('std 10000, 68% of |x| > 4096', '0'): (3542, 2497, 6546),
}


def envelope():
    rng = np.random.RandomState(1)
    K = ENVELOPE_K
    table = []
    for e in range(-10, 11, 2):
        s = 2.0 ** e
        for ratio in (0, 1, 16, 256):
            x = s * rng.standard_normal(K) + ratio * s
            if np.abs(x).max() > 60000:
                continue
            table.append((f"std 2^{e}", f"{ratio}", *envelope_row(x)))
    for c in (0.1, 7.0, 1000.0):
        table.append((f"constant {c}", "-", *envelope_row(np.full(K, c))))
    for s in (1000.0, 3000.0, 10000.0):
        x = np.clip(s * rng.standard_normal(K), -60000, 60000)
        table.append((f"std {s:g}, {(np.abs(x) > 4096).mean():.0%} of |x| > 4096", "0", *envelope_row(x)))
    return table


def test_format_envelope():
    with np.errstate(over="ignore", invalid="ignore"):
        table = envelope()
    print(f"\nLayerNorm staging vs float64, K {ENVELOPE_K}, gamma 1, beta 0")
    print("| row | abs(mean) / std | max ulps | median ulps | max abs error in ulp(1) |")
    for r in table:
        print(f"| {r[0]} | {r[1]} | {r[2]:.3g} | {r[3]:.3g} | {r[4]:.3g} |")
    got = {(a, b): r for a, b, *r in table}
    assert set(got) == set(ENVELOPE)
    for key, want in ENVELOPE.items():
        g = np.array(got[key])
        w = np.array(want)
        assert ((np.isinf(g) & np.isinf(w)) | np.isclose(g, w, rtol=0.01, atol=1e-6)).all(), (key, tuple(g), want)
