"""The decode step's four Conv1D phases (csrc/decode_engine.cu gemm_phase<R>) restated for tests: the partition of one
(CTA, Conv1D), a float64 Conv1D of the operands the kernel sees, the admissible fp16 outputs under a rigorous bound, and
a numpy emulation of the kernel's summation order.

TEST INFRASTRUCTURE ONLY (only tests/ may import it).  numpy.

Partition (restated exactly from gemm_phase and jk_prior_plan):
    columns     unit u = CTA c / KS owns the 8-column groups [g0, g0 + ncg) of each Conv1D (the plan's `cols`); rank
                r = c % KS multiplies the K slice [r K / KS, (r + 1) K / KS), nkk = K / KS / 16 k-steps
    ring        kpc = kpc_of(ncg) k-steps per slot, nslots = ceil(nkk / kpc); in_order = nslots > the plan's ring_slots
    dealing     contiguous runs (k-step i -> warp i * 8 / nkk) when nkk >= 8, one k-step per warp when nkk < 8, and in
                in_order phases whole slots round robin (slot s -> warp s mod 8); every warp walks the slots in order
    nwarp       min(8, nslots) in_order, else min(8, nkk): the warps whose tiles the cross-warp reduction reads
    reduction   per rank: the nwarp tiles summed in warp order (fp32, from 0); KS > 1: the KS rank partials, exchanged as
                LL words, summed in rank order (fp32, from 0); KS = 1: the warp sum is the Conv1D sum
    epilogue    ppc = 4 ncg / KS column pairs per CTA, rank r finishes pairs [r ppc, (r + 1) ppc) of its unit;
                two_rows (ppc <= 16): lane & 15 = pair, rows 2 warp + (lane >> 4) + 16 i; else lane = pair, rows warp + 8 i
                y = fp16(fp32(s + b)); qkv: y; fc: quick_gelu16(y); proj / proj2: fp16(fp32(x + y))

Operands: weights fp16 as pack_gemm_kernel rounds them (__float2half_rn of fp32, or the fp16 value), biases fp32 of
fp16 (round_bias_kernel), activations the fp16 rows the staging writes (oracle.decode_stats.staged for the LayerNorm
phases, the previous phase's fp16 outputs otherwise).  Products of two fp16 values are exact in float64, and the float64
sums of at most 4800 of them are within K 2^-53 sum |a w| < 2^-40 sum |a w| of the exact sum; that margin is charged.

Bound on |fl(s + b) - (s64 + b)| (`bound`), per output element, following the kernel's order:
  (1) MMA (m16n8k16, fp32 accumulate): one k-step of one warp adds 16 exact fp16 x fp16 products to the accumulator C.
      How mma.sync rounds inside that sum is not documented for Hopper.  What is published for earlier tensor cores
      (Fasi, Higham, Mikaitis, Pranesh 2021) is an alignment of the addends to the largest exponent with the bits past
      the 24th truncated, then a normalisation; that loses at most one unit in the 24th bit of the largest addend per
      addend and one of the result.  The bound charges twice that, u = 2^-22 per addend instead of 2^-23, so that a
      path keeping one bit fewer is covered too, and it charges every addend at the larger of |C| and the k-step's sum
      of |products| (which is at least its largest product):  e_t <= 17 u (|C_t| + d_t + Q_t), Q_t = sum |a w| of the
      k-step, C_t the exact running sum in the warp's k-step order and d_t the error accumulated so far.  This term is
      deliberately conservative; it is not fitted to what a card happens to return.
  (2) the warp's k-steps in sequence: (1) accumulated along the dealt order (exact partial sums C_t, computed here).
  (3) the cross-warp sum in warp order from 0: adding to 0 is exact, then one fp32 round-to-nearest add per warp,
      2^-24 (|exact running sum| + accumulated error) each.
  (4) the rank sum in rank order from 0 (KS > 1): the same, one add per rank after the first.
  (5) the bias add: 2^-24 (|s + b| + accumulated error).
The admissible outputs (`admissible`) are then every fp16 value that rounds from [s64 + b - bound, s64 + b + bound]
(rounding is monotone): fp16(s64 + b), and its neighbour when s64 + b lies within the bound of a rounding midpoint.
Term (1) makes the bound wide where a sum cancels (an output near 0 against sum |a w|): there the range holds several
fp16 values, and the tests report how many.

Exact probes: when every activation and weight lies on a grid 2^-ea, 2^-ew and sum |a w| + |b| < 2^24 2^-(ea + ew),
every partial sum in any order, inside or outside an MMA, is an fp32 value: the kernel must return fp16(s64 + b) bit for
bit.  `exact_in_fp32` checks that condition for the probes' operands."""
import numpy as np

from oracle.decode_stats import quick_gelu16

NWARPS = 8
U_MMA = 2.0 ** -22             # (1): twice the per-addend loss of a 24-bit alignment with truncation
U_ADD = 2.0 ** -24             # fp32 round to nearest
F64_MARGIN = 2.0 ** -40


def kpc_of(ncg):
    return 64 if ncg == 1 else 32 if ncg == 2 else 16 if ncg <= 4 else 8


class Phase:
    """the partition of one (CTA, Conv1D) with ncg column groups: K slice, ring slots, warp dealing, epilogue layout.
    mutate (planted faults for the tests that show the checks catch them): "in_order_drop" (the last slot of warp 0 is
    skipped), "in_order_twice" (warp 1 also multiplies warp 0's first slot)"""

    def __init__(self, K, KS, ncg, ring_slots, mutate=None):
        self.K, self.KS, self.ncg = K, KS, ncg
        self.Ks = K // KS
        self.nkk = self.Ks // 16
        self.kpc = kpc_of(ncg)
        self.nslots = -(-self.nkk // self.kpc)
        self.in_order = self.nslots > ring_slots
        self.nwarp = min(NWARPS, self.nslots) if self.in_order else min(NWARPS, self.nkk)
        self.ppc = (ncg * 4) // KS
        self.two_rows = self.ppc <= 16
        self.steps = [self._deal(w) for w in range(NWARPS)]
        if mutate == "in_order_drop":
            assert self.in_order
            mine = [s for s in range(self.nslots) if s % NWARPS == 0]
            last = mine[-1] * self.kpc
            self.steps[0] = [k for k in self.steps[0] if not (last <= k < last + self.kpc)]
        elif mutate == "in_order_twice":
            assert self.in_order
            self.steps[1] = sorted(self.steps[1] + list(range(0, min(self.kpc, self.nkk))))

    def _deal(self, warp):
        nkk, kpc = self.nkk, self.kpc
        if nkk >= 8:
            k_lo, k_hi = (warp * nkk) >> 3, ((warp + 1) * nkk) >> 3
        else:
            k_lo, k_hi = min(warp, nkk), min(warp + 1, nkk)
        out = []
        for slot_i, kk0 in enumerate(range(0, nkk, kpc)):
            a, b = max(kk0, k_lo), min(kk0 + kpc, nkk, k_hi)
            if self.in_order:
                a, b = kk0, (min(kk0 + kpc, nkk) if slot_i % NWARPS == warp else kk0)
            out += range(a, b)
        return out

    def finished(self, B):
        """(rank, warp, lane, row, pair inside the unit) of every output pair the epilogue writes"""
        out = []
        for r in range(self.KS):
            for warp in range(NWARPS):
                for lane in range(32):
                    pl = (lane & 15) if self.two_rows else lane
                    if pl >= self.ppc:
                        continue
                    b0, step = (2 * warp + (lane >> 4), 16) if self.two_rows else (warp, 8)
                    for b in range(b0, B, step):
                        out.append((r, warp, lane, b, r * self.ppc + pl))
        return out


def unit_groups(cols_l_gi):
    """{ncg: [column indices]} of one Conv1D of one layer, from the plan's [U, 2] (g0, ncg) records"""
    out = {}
    for g0, ncg in cols_l_gi:
        if ncg:
            out.setdefault(int(ncg), []).append(np.arange(8 * g0, 8 * (g0 + ncg)))
    return {k: np.concatenate(v) for k, v in out.items()}


# ---- operands ------------------------------------------------------------------------------------------------------
def weights16(w):
    """the fp16 weights pack_gemm_kernel streams (fp32 rounded to nearest even, fp16 as is)"""
    return np.asarray(w).astype(np.float16)


def bias32(b):
    """round_bias_kernel: fp32 of the fp16-rounded bias"""
    return np.asarray(b).astype(np.float16).astype(np.float32)


def conv64(A, W, b=None):
    """s64 + b in float64 of fp16 activations A [B, K] and fp16 weights W [K, N]"""
    s = np.asarray(A, np.float64) @ np.asarray(W, np.float64)
    return s if b is None else s + np.asarray(b, np.float64)


def exact_in_fp32(A, W, b):
    """True if every partial sum of A . W + b, in any order, is an fp32 value (module docstring)"""
    def grid(v):                       # the smallest e with every value a multiple of 2^-e (fp16 / fp32 values)
        v = np.abs(np.asarray(v, np.float64))
        v = v[v != 0]
        if v.size == 0:
            return -64
        n = (v * 2.0 ** 40).astype(np.int64)
        assert (n == v * 2.0 ** 40).all() and v.max() < 2.0 ** 22
        return 40 - int(np.log2(np.bitwise_and(n, -n)).min())
    ea, ew, eb = grid(A), grid(W), grid(b)
    if eb > ea + ew:
        return False
    mag = np.abs(np.asarray(A, np.float64)) @ np.abs(np.asarray(W, np.float64)) + np.abs(np.asarray(b, np.float64))
    return bool(mag.max() < 2.0 ** (24 - ea - ew))


# ---- the bound -----------------------------------------------------------------------------------------------------
def _rank_partials(A, W, phase, r, mma_err=True):
    """per warp: (exact partial sums, accumulated MMA error) of rank r's K slice, [B, ncols] each"""
    Ks = phase.Ks
    out = []
    for w in range(phase.nwarp):
        C = np.zeros((A.shape[0], W.shape[1]))
        d = np.zeros_like(C)
        for kk in phase.steps[w]:
            sl = slice(r * Ks + 16 * kk, r * Ks + 16 * kk + 16)
            a, ww = A[:, sl], W[sl]
            if mma_err:
                Q = np.abs(a) @ np.abs(ww)
                d = d + 17 * U_MMA * (np.abs(C) + d + Q)
            C = C + a @ ww
        out.append((C, d))
    return out


def _ordered_sum(parts):
    """exact sum and error bound of fp32 partials (value, error) added in order starting from 0"""
    s, d = parts[0][0].copy(), parts[0][1].copy()
    for v, e in parts[1:]:
        s = s + v
        d = d + e
        d = d + U_ADD * (np.abs(s) + d)
    return s, d


def bound(A, W, b, phase):
    """(s64 + b, bound) of the columns of units with this phase's ncg: A [B, K] fp16, W [K, ncols] fp16, b [ncols] fp32
    (module docstring)"""
    A = np.asarray(A, np.float64)
    W = np.asarray(W, np.float64)
    ranks = [_ordered_sum(_rank_partials(A, W, phase, r)) for r in range(phase.KS)]
    s, d = _ordered_sum(ranks)
    sb = s + np.asarray(b, np.float64)
    d = d + U_ADD * (np.abs(sb) + d)
    d = d + F64_MARGIN * (np.abs(A) @ np.abs(W) + np.abs(b))
    return sb, d


def conv_bound(A, W, b, groups, phases):
    """(s64 + b, bound) of a whole Conv1D [B, N]: groups {ncg: column indices}, phases {ncg: Phase}"""
    N = W.shape[1]
    sb = np.full((A.shape[0], N), np.nan)
    bd = np.full_like(sb, np.nan)
    for ncg, idx in groups.items():
        sb[:, idx], bd[:, idx] = bound(A, W[:, idx], b[idx], phases[ncg])
    return sb, bd


# ---- admissible outputs --------------------------------------------------------------------------------------------
def f16(x):
    return np.asarray(x, np.float64).astype(np.float16)


def _steps(v, n):
    for _ in range(abs(n)):
        v = np.nextafter(v, np.float16(np.sign(n) * np.inf))
    return v


def admissible(kind, sb, bd, x=None, enum=8):
    """(lo, hi, nearest): the admissible phase outputs of every element lie in [lo, hi] (fp16 arrays), nearest is the
    output of fp16(s64 + b).  y ranges over the fp16 values of [sb - bd, sb + bd] (rounding is monotone); qkv: y;
    fc: quick_gelu16(y), each of up to `enum` candidates with its fp16 neighbours where the oracle flags the device's
    expf as able to round the other way, and a longer run of candidates (the bound passes `enum` fp16 ulps: an output
    near 0, whose sum cancelled) only on [-1/2, inf), where quick_gelu is increasing, from the end points widened by
    4 fp16 ulps (the roundings inside quick_gelu16 are not monotone by themselves); proj / proj2: fp16(fp32(x + y)),
    increasing in y.  Also returns the number of y candidates per element."""
    near, lo, hi = f16(sb), f16(sb - bd), f16(sb + bd)
    n = np.ones(near.shape, np.int64)
    cur = near
    while True:                                         # count the candidates, up to enum + 1
        nxt = _steps(cur, 1)
        more = (nxt.astype(np.float64) <= hi.astype(np.float64)) & (n <= enum)
        if not more.any():
            break
        cur, n = np.where(more, nxt, cur), n + more
    cur = near
    while True:
        nxt = _steps(cur, -1)
        more = (nxt.astype(np.float64) >= lo.astype(np.float64)) & (n <= enum)
        if not more.any():
            break
        cur, n = np.where(more, nxt, cur), n + more
    if kind == "fc":
        gn, _ = quick_gelu16(near)
        glo, ghi = np.full(near.shape, np.inf), np.full(near.shape, -np.inf)
        cur = lo
        for _ in range(enum):
            valid = cur.astype(np.float64) <= hi.astype(np.float64)
            g, nr = quick_gelu16(cur)
            gm, gp = np.where(nr, _steps(g, -1), g), np.where(nr, _steps(g, 1), g)
            glo = np.where(valid, np.minimum(glo, gm.astype(np.float64)), glo)
            ghi = np.where(valid, np.maximum(ghi, gp.astype(np.float64)), ghi)
            cur = _steps(cur, 1)
        long = cur.astype(np.float64) <= hi.astype(np.float64)
        if long.any():
            assert (lo[long] >= -0.5).all(), "a long run of candidates where quick_gelu is not increasing"
            glo = np.where(long, np.minimum(glo, _steps(quick_gelu16(lo)[0], -4).astype(np.float64)), glo)
            ghi = np.where(long, np.maximum(ghi, _steps(quick_gelu16(hi)[0], 4).astype(np.float64)), ghi)
        near, lo, hi = gn, f16(glo), f16(ghi)
    if x is not None:
        near, lo, hi = residual(x, near), residual(x, lo), residual(x, hi)
    return lo, hi, near, n


def residual(x, y):
    """EPI_PROJ / EPI_PROJ2: fp16(fp32(x + y)), x and y fp16 values (a double rounding, as the reference)"""
    return (np.asarray(x, np.float16).astype(np.float32) + np.asarray(y, np.float16).astype(np.float32)).astype(np.float16)


def in_interval(got, lo, hi):
    got = np.asarray(got, np.float64)
    return (np.asarray(lo, np.float64) <= got) & (got <= np.asarray(hi, np.float64))


# ---- emulation of the kernel's order -------------------------------------------------------------------------------
def _mma_rn(C, a, w):
    """one m16n8k16 with one round-to-nearest of (C + sum of the exact products) to fp32"""
    return (C.astype(np.float64) + a @ w).astype(np.float32)


def _mma_trunc(C, a, w):
    """one m16n8k16 as the published model of earlier tensor cores: every addend aligned to the largest exponent and
    truncated to 24 bits, summed, the sum truncated to 24 bits (toward zero)"""
    prods = a[:, :, None] * w[None, :, :]                                  # [B, 16, n] exact
    add = np.concatenate([C.astype(np.float64)[:, None, :], prods], axis=1)
    mx = np.abs(add).max(1, keepdims=True)
    _, e = np.frexp(np.where(mx > 0, mx, 1.0))
    q = np.ldexp(1.0, e - 24)                                              # the 24th bit of the largest addend
    s = (np.trunc(add / q) * q).sum(1)
    _, es = np.frexp(np.where(s != 0, s, 1.0))
    qs = np.ldexp(1.0, es - 24)
    return (np.trunc(s / qs) * qs).astype(np.float32)


def emulate(A, W, b, phase, mma="rn", mutate=None, other=None):
    """gemm_phase's arithmetic for the columns of one ncg group (A [B, K] fp16, W [K, ncols] fp16, b [ncols] fp32) in
    its order: fp32 warp accumulators over the dealt k-steps, the cross-warp sum, the rank sum, the bias add, then
    y = fp16(fp32(s + b)).  Planted faults (mutate): "rank_missing" (rank KS - 1's partial is not added),
    "rank_stale" (rank KS - 1's partial is read from the previous Conv1D's exchange: `other`, [B, ncols] fp32),
    "pair_no_rank_offset" (pr = pl: every rank finishes rank 0's pairs, the other pairs are never written: returned
    NaN), "bias_next_pair" (the bias of the next column pair), "rows_tile0" (rows 16-31 multiply the A rows of tile 0)."""
    f32 = np.float32
    A = np.asarray(A, np.float64)
    W = np.asarray(W, np.float64)
    if mutate == "rows_tile0":
        A = A.copy()
        A[16:32] = A[0:min(16, A.shape[0] - 16)]
    mma_f = _mma_rn if mma == "rn" else _mma_trunc
    Bn, ncols = A.shape[0], W.shape[1]
    ranks = []
    for r in range(phase.KS):
        tiles = []
        for w in range(phase.nwarp):
            C = np.zeros((Bn, ncols), f32)
            for kk in phase.steps[w]:
                sl = slice(r * phase.Ks + 16 * kk, r * phase.Ks + 16 * kk + 16)
                C = mma_f(C, A[:, sl], W[sl])
            tiles.append(C)
        s = np.zeros((Bn, ncols), f32)
        for t in tiles:
            s = (s + t).astype(f32)
        ranks.append(s)
    if mutate == "rank_missing":
        ranks = ranks[:-1]
    elif mutate == "rank_stale":
        ranks = ranks[:-1] + [np.asarray(other, f32)]
    s = np.zeros((Bn, ncols), f32)
    for v in ranks:
        s = (s + v).astype(f32)
    bb = np.asarray(b, f32)
    if mutate == "bias_next_pair":
        bb = np.concatenate([bb[2:], bb[:2]])          # within a group of units: the pair after, wrapping
    y = (s + bb).astype(f32).astype(np.float16)
    if mutate == "pair_no_rank_offset":
        y = y.astype(np.float32)
        cols_in_unit = 8 * phase.ncg
        for u0 in range(0, ncols, cols_in_unit):
            y[:, u0 + 2 * phase.ppc: u0 + cols_in_unit] = np.nan
        y = y.astype(np.float16)
    return y


# ---- probe operands ------------------------------------------------------------------------------------------------
def grid_weights(rng, K, N, scale=2.0 ** -3):
    """sparse weights on the grid {-7..7} scale, [K, N] float32: column n has one nonzero in every k-step kk = n mod d
    (d <= 8, about 40 k-steps per column), at row (5 n + 3 kk) mod 16 of the k-step, so every k-step of every unit (8
    columns or more) meets a nonzero weight and a dropped or repeated k-step moves some column"""
    nkk = K // 16
    d = min(8, max(1, -(-nkk // 40)))
    w = np.zeros((K, N), np.float32)
    n = np.arange(N)
    for kk in range(nkk):
        cols = n[n % d == kk % d]
        rows = 16 * kk + (5 * cols + 3 * kk) % 16
        mag = rng.integers(1, 8, cols.size) * np.where(rng.random(cols.size) < 0.5, -1.0, 1.0)
        w[rows, cols] = mag * scale
    return w


def grid_bias(rng, N, scale=2.0 ** -3):
    return (rng.integers(-7, 8, N) * scale).astype(np.float32)


def grid_rows(rng, B, W):
    """grid-valued residual rows x (multiples of 1/4 in [-2, 2], no row constant): fp16 values as float32"""
    x = rng.integers(-8, 9, (B, W)).astype(np.float32) / 4
    x[:, :2] = [1.0, -1.0]
    return x


def exact_ln(rng, W, lo=1.0, hi=1.25, gscale=2.0 ** -5):
    """LayerNorm gamma / beta whose staged rows stay in +-[lo - 0.5, hi + 0.5] with fp16 values of 11 bits at most
    below 2^-11 (|x - mean| rstd <= 4 on the probes' rows): small gamma, beta of magnitude about 1"""
    gamma = (rng.integers(1, 5, W) * gscale * np.where(rng.random(W) < 0.5, -1, 1)).astype(np.float32)
    beta = ((lo + rng.integers(0, 5, W) * (hi - lo) / 4) * np.where(rng.random(W) < 0.5, -1, 1)).astype(np.float32)
    return gamma, beta


def identity_gelu_ln(rng, W):
    """LN1 gamma / beta whose staged values are 0 or in [8, 16), where quick_gelu16 is the identity: a quarter of the
    columns gamma = beta = 0, the rest beta in {10 .. 13}, |gamma| <= 2^-2"""
    zero = rng.random(W) < 0.25
    gamma = np.where(zero, 0, rng.integers(1, 3, W) * 2.0 ** -3 * np.where(rng.random(W) < 0.5, -1, 1))
    beta = np.where(zero, 0, rng.integers(10, 14, W)).astype(np.float32)
    return gamma.astype(np.float32), beta
