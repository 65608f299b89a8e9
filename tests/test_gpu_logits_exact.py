"""GPU: the decode engine's logits against a float64 product, elementwise, in every logits plan, and the fp32 SGEMM
jk_f32_linear against float64.

The logits are linear in the final residual stream h, and jk_prior_step returns h (h_out: fp32 copies of the fp16 values
the logits product multiplies) in the same call as the logits.  A float64 product on the CPU is then an exact reference:
    exact = y . x_out^T (+ bias)        y = h, or h + x_cond where the FMA product adds x_cond itself
    split = h . (hi + lo)^T (+ bias)    hi = fp16(x_out), lo = fp16(x_out - hi), as pack_logits_kernel forms them
and the two bounds below are elementwise:
    tensor-core GEMM:  |got - split| <= acc                and  |got - exact| <= acc + |split - exact|
    fp32 FMA product:  |got - exact| <= acc
|split - exact| is the representation error of hi + lo: with x_out at the reference's scale, N(0, 0.02^2), nearly every
lo half is an fp16 subnormal (absolute step 2^-24).

The bound acc.  Every product the engine sums is exact in fp32 (fp16 x fp16 on the tensor cores; the FMA path rounds
once per fma), so the error is that of the fp32 additions.  Each errs by at most 2u times the partial sum it rounds
(u = 2^-24; 2u because the tensor cores' accumulation truncates).  The n products p = h o x_v have random signs, so a
partial sum over m of them is about ||p||_2 sqrt(m / n) in size.  On the GEMM a product meets about 20 roundings on its
way to a logit (its warp's k-steps, the 8 warps' tiles, the K-split ranks).  With every rounding at its largest, all of
one sign, and every partial sum at three standard deviations, they add up to about 25 u ||p||_2 at W = 2048 (K split 4)
and 27 u ||p||_2 at W = 1152 (K split 2).  The FMA path sums W / 32 products per lane, then a 5-level shuffle tree, with
a smaller error.  The bound is
    acc(b, v) = 2 u sqrt(n) ||p||_2 + u |exact|     (n = 2 W products on the GEMM, W on the FMA path)
(128 u ||p||_2 at W = 2048, 96 u ||p||_2 at W = 1152), plus, where they apply, u sum_k |y_k x_vk| for rounding
y = h + x_cond to fp32 and gamma_W sum_k |x_cond,k x_vk| for a logit bias that jk_f32_linear computed.  On an H100 the
largest err / acc is 0.31, at W = 1152 and 32 rows: close to the one-sign estimate, because truncation errors share the
sign of the partial sum they cut.
A worst-case bound, 2 W u sum |p|, would be about as large as the error of dropping lo; acc is not: in every GEMM case
the test asserts that the error of hi alone, |h . hi^T - exact|, is at least 10 acc at the median element, so a lost or
misread lo half cannot pass."""
import json

import numpy as np
import pytest
import torch

from jukebox_b200 import _lib
from oracle.synth import synth_state_dict, synth_tensor
from test_logits_plan_matrix_cpu import CASES, N_CTX, plan_info, set_case_env

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
STEPS = 3               # positions stepped per run


def gamma(k):
    """the classical bound of k fp32 roundings in sequence: |error| <= gamma_k * sum |terms|"""
    return k * U / (1 - k * U)


class XOut:
    """x_out [bins, W] at the reference's scale, N(0, 0.02^2), with planted entries in every row: three whose hi half is an
    fp16 subnormal (below 2^-14), one near 1, three exact zeros.  Its fp16 halves are formed as pack_logits_kernel forms
    them: x - hi is exact in fp32, then rounded to fp16 (numpy rounds to nearest even, subnormals included)."""

    def __init__(self, bins, width, rng):
        x = (rng.standard_normal((bins, width)) * 0.02).astype(np.float32)
        r, cols = np.arange(bins)[:, None], rng.randint(0, width, (bins, 7))
        sign = lambda k: np.where(rng.random_sample((bins, k)) < 0.5, -1.0, 1.0)
        x[r, cols[:, 0:3]] = sign(3) * rng.uniform(2.0 ** -24, 2.0 ** -14, (bins, 3))
        x[r, cols[:, 3:4]] = sign(1) * rng.uniform(0.9, 1.1, (bins, 1))
        x[r, cols[:, 4:7]] = 0.0
        hi = x.astype(np.float16)
        lo = (x - hi.astype(np.float32)).astype(np.float16)
        self.x = x
        self.x64 = x.astype(np.float64)
        self.abs = np.abs(self.x64)
        self.sq = self.x64 ** 2
        self.hi = hi.astype(np.float64)
        self.split = self.hi + lo.astype(np.float64)
        self.sq_split = self.hi ** 2 + lo.astype(np.float64) ** 2
        nz = lo != 0
        self.lo_subnormal = float((np.abs(lo[nz]) < 2.0 ** -14).mean())


def check_logits(got, h, xo, gemm, cond=None, bias=None):
    """Assert the bounds of the module docstring for one run.  got, h: [rows, bins], [rows, W] in float64, one row per
    (position, sample).  gemm: the tensor-core product ran, else the FMA product.  cond: the x_cond row of each
    (position, sample): the FMA path adds it to y; on the GEMM path it is what jk_f32_linear made the logit bias from.
    bias: a synthetic logit bias [rows, bins] (GEMM path).  Returns (statistics, the bound on |got - exact|, exact)."""
    W = h.shape[1]
    y = h if (gemm or cond is None) else h + cond
    exact = y @ xo.x64.T
    extra = 0.0
    if gemm:
        n, pn = 2 * W, np.sqrt((h * h) @ xo.sq_split.T)
        split, hi_only = h @ xo.split.T, h @ xo.hi.T
        add = bias
        if bias is None and cond is not None:
            add = cond @ xo.x64.T                                   # (h + x_cond) . x_out^T = h . x_out^T + bias
            extra = gamma(W) * (np.abs(cond) @ xo.abs.T)            # the bias's own fp32 product
        if add is not None:
            exact, split, hi_only = exact + add, split + add, hi_only + add
    else:
        n, pn = W, np.sqrt((y * y) @ xo.sq.T)
        if cond is not None:
            extra = U * (np.abs(y) @ xo.abs.T)                      # y = h + x_cond rounded to fp32
    acc = 2 * U * np.sqrt(n) * pn + U * np.abs(exact) + extra

    def require(err, bound, what):
        ratio = err / bound
        i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        assert ratio[i] <= 1.0, (f"{what}: |err| {err[i]:.3e} > bound {bound[i]:.3e} at (row {i[0]}, v {i[1]}): "
                                 f"got {got[i]!r} exact {exact[i]!r}; {(ratio > 1).sum()} of {ratio.size} elements over")
        return float(ratio[i])

    st = {}
    if gemm:
        rep = np.abs(split - exact)
        st["err_over_bound"] = require(np.abs(got - split), acc, "logits GEMM vs h . (hi + lo)")
        tol = acc + rep
        require(np.abs(got - exact), tol, "logits GEMM vs h . x_out")
        st["rep_err"] = float(rep.max())
        st["rep_over_range"] = float(rep.max() / (exact.max() - exact.min()))
        st["hi_only_over_bound"] = float(np.median(np.abs(hi_only - exact) / acc))
    else:
        tol = acc
        st["err_over_bound"] = require(np.abs(got - exact), acc, "FMA logits vs y . x_out")
    return st, tol, exact


class CaseData:
    """inputs of one case, shared by its engines: weights from oracle/synth.py, tokens, y_cond, x_cond, logit biases"""

    def __init__(self, case, seed):
        from jukebox_b200.transformer.transformer import Transformer
        W, bins = case.width, case.bins
        tr = Transformer(W, N_CTX, case.heads, 1, mask=True, attn_order=0)
        sd = synth_state_dict([(k, tuple(v.shape)) for k, v in tr.state_dict().items()], seed)
        tr.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
        self.block = tr.cuda().eval()._attn_mods[0]
        rng = np.random.RandomState(seed)
        self.xo = XOut(bins, W, rng)
        cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.x_out = cuda(self.xo.x)
        self.x_emb = cuda(synth_tensor("x_emb.weight", (bins, W), seed))
        self.pos_emb = cuda(synth_tensor("pos_emb.pos_emb", (N_CTX, W), seed))
        self.tokens = cuda(rng.randint(0, bins, (32, N_CTX)).astype(np.int64))
        self.y_cond = cuda((rng.standard_normal((32, W)) * 0.5).astype(np.float32))
        self.xc_pos = cuda((rng.standard_normal((32, N_CTX, W)) * 0.5).astype(np.float32))
        self.xc_one = cuda((rng.standard_normal((32, 1, W)) * 0.5).astype(np.float32))
        self.rng = rng
        self.lb_one = self.lb_pos = None

    def make_biases(self, scale):
        """a random row of the logits' own magnitude for every (sample, position): a bias read from the wrong row, position
        or column lands far outside the bound, and at this size fp32 keeps the precision the bound relies on"""
        bins = self.xo.x.shape[0]
        self.lb_one = torch.from_numpy((self.rng.standard_normal((32, 1, bins)) * scale).astype(np.float32)).cuda()
        self.lb_pos = torch.from_numpy((self.rng.standard_normal((32, N_CTX, bins)) * scale).astype(np.float32)).cuda()


def step_run(eng, d, n, x_cond, logit_bias):
    """positions 0 .. STEPS-1 of n samples, the logits written into a NaN-filled buffer in the get_preds layout
    [rows, n_ctx, bins] (logits_bstride = n_ctx * bins, logits_tstride = bins) with more rows than the kernel has.
    Returns (logits [STEPS * n, bins], h_out [STEPS * n, W]) in float64, position-major."""
    bins = d.xo.x.shape[0]
    buf = torch.full(((16 if n <= 16 else 32) + 1, N_CTX, bins), float("nan"), device="cuda")
    eng.reset(0)
    hs = []
    for _ in range(STEPS):
        h = torch.empty(n, d.y_cond.shape[1], device="cuda")
        eng.step(n, tokens=d.tokens[:n], y_cond=d.y_cond[:n], x_cond=x_cond, h_out=h, logits=buf, logits_tstride=bins,
                 logit_bias=logit_bias)
        hs.append(h)
    torch.cuda.synchronize()
    # no write outside [b < n, t < STEPS, v < bins]: not the padded last column, not rows n .. 31 of the 32-row kernel
    assert bool(torch.isnan(buf[n:]).all()) and bool(torch.isnan(buf[:, STEPS:]).all()), "logits written out of range"
    got = buf[:n, :STEPS].transpose(0, 1).reshape(STEPS * n, bins).double().cpu().numpy()
    assert np.isfinite(got).all()
    return got, torch.cat(hs).double().cpu().numpy()


def rows_of(a, n):
    """the row of an [n, 1 or n_ctx, *] x_cond or logit bias for every (position, sample) of a run, position-major"""
    a = a[:n].double().cpu().numpy()
    return np.concatenate([a[:, t if a.shape[1] > 1 else 0] for t in range(STEPS)])


@pytest.mark.parametrize("name", list(CASES))
def test_logits_exact(name, monkeypatch):
    from jukebox_b200.engine import DecodeEngine
    from jukebox_b200.transformer import f32
    case = CASES[name]
    set_case_env(monkeypatch, case)           # read when the engine is planned
    sms = _lib.sm_count()
    d = CaseData(case, 3)
    W, bins = case.width, case.bins
    report = dict(case=name, sms=sms, lo_subnormal=round(d.xo.lo_subnormal, 4), runs=[])
    worst, hi_only, rep, rep_rel, hmax = 0.0, [], 0.0, 0.0, 0.0
    engines = {}
    for mb, n in case.runs:
        if mb not in engines:
            engines.clear()
            eng = DecodeEngine(width=W, depth=1, heads=case.heads, n_state=W // 4, mlp_width=W, n_ctx=N_CTX, blocks=0,
                               attn_funcs=[0], bins=bins, max_batch=mb)
            eng.load_layer(0, d.block)
            eng.set_embeddings(x_emb=d.x_emb, pos_emb=d.pos_emb, x_out=d.x_out)
            info = plan_info(case, mb, sms)
            assert eng.has_logits_gemm == (info.logits_passes > 0)
            if sms == 132:                     # the plans the CPU test pins
                assert (info.k_split, info.logits_passes) == case.plans[mb]
            engines[mb] = (eng, info)
        eng, info = engines[mb]
        gemm = info.logits_passes > 0
        # bias modes: none; a synthetic bias [n, 1, bins] (tstride 0) and [n, n_ctx, bins]; x_cond without a bias (the
        # FMA product of h + x_cond, also on a GEMM engine); the real bias, x_cond . x_out^T from jk_f32_linear.  An FMA
        # engine ignores a bias it is given.
        modes = ["none", "bias_one", "bias_pos", "xcond", "real"] if gemm else ["none", "xcond", "bias_ignored"]
        run_worst = 0.0
        for mode in modes:
            xc = {"none": None, "bias_one": d.xc_one, "bias_pos": d.xc_pos, "xcond": d.xc_pos, "real": d.xc_pos,
                  "bias_ignored": d.xc_one}[mode]
            xc = None if xc is None else xc[:n]
            lb = {"bias_one": d.lb_one, "bias_pos": d.lb_pos, "bias_ignored": d.lb_one}.get(mode)
            if mode == "real":
                lb = f32.linear_nk(xc.reshape(n * N_CTX, W), d.x_out).view(n, N_CTX, bins)
            got, h = step_run(eng, d, n, xc, None if lb is None else lb[:n])
            on_gemm = gemm and mode != "xcond"
            cond = None if xc is None else rows_of(xc, n)
            bias = rows_of(lb, n) if mode in ("bias_one", "bias_pos") else None
            st, tol, exact = check_logits(got, h, d.xo, on_gemm, cond=cond, bias=bias)
            run_worst = max(run_worst, st["err_over_bound"])
            hmax = max(hmax, float(np.abs(h).max()))
            if on_gemm:
                rep, rep_rel = max(rep, st["rep_err"]), max(rep_rel, st["rep_over_range"])
                if mode != "real":
                    hi_only.append(st["hi_only_over_bound"])
                    assert st["hi_only_over_bound"] >= 10, (mode, st)      # the bound sees a lost lo half
            if mode == "none":
                if d.lb_one is None:
                    d.make_biases(float(exact.std()))
                # the other route to the same logits (get_preds mixes both): jk_f32_linear on the step's h_out
                lin = f32.linear_nk(torch.from_numpy(h).float().cuda(), d.x_out).double().cpu().numpy()
                tol_lin = tol + gamma(W) * (np.abs(h) @ d.xo.abs.T)
                assert (np.abs(got - lin) <= tol_lin).all(), float((np.abs(got - lin) / tol_lin).max())
        worst = max(worst, run_worst)
        report["runs"].append([mb, n, info.k_split, info.logits_passes, round(run_worst, 4)])
    report.update(worst_err_over_bound=round(worst, 4), max_abs_h=round(hmax, 2))
    if hi_only:
        report.update(hi_only_over_bound_min=round(min(hi_only), 1), rep_err=float(f"{rep:.3e}"),
                      rep_err_over_range=float(f"{rep_rel:.3e}"))
    print(json.dumps(report))


# ---- jk_f32_linear: y[M, N] = x[M, K] . w + b in fp32 (logit bias, prefilled get_preds logits, prime logits) ----------
def f32_linear(x, w, b, w_is_nk):
    M, K = x.shape
    N = w.shape[0] if w_is_nk else w.shape[1]
    y = torch.empty(M, N, device=x.device)
    _lib.check(_lib.lib().jk_f32_linear(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(y), M, N, K, int(w_is_nk),
                                        _lib.stream_ptr()))
    return y


def check_linear(y, x, w, b, w_is_nk):
    """K fmas in sequence, then the bias: |y - x . w - b| <= gamma_{K+1} (sum_k |x_k w_k| + |b|)"""
    wk = w.T if w_is_nk else w
    ref = x @ wk + (0.0 if b is None else b)
    scale = np.abs(x) @ np.abs(wk) + (0.0 if b is None else np.abs(b))
    ratio = np.abs(y - ref) / (gamma(x.shape[1] + 1) * scale)
    assert ratio.max() <= 1.0, float(ratio.max())
    return float(ratio.max())


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("w_is_nk", [0, 1])
@pytest.mark.parametrize("M, N, K", [(77, 131, 45), (1, 2127, 2048), (130, 70, 1920), (64, 128, 32)])
def test_f32_linear_against_float64(M, N, K, w_is_nk, bias):
    rng = np.random.RandomState(M * N + K + 2 * w_is_nk + bias)
    x = rng.standard_normal((M, K)).astype(np.float32)
    w = (rng.standard_normal((N, K) if w_is_nk else (K, N)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32) if bias else None
    y = f32_linear(torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), None if b is None else torch.from_numpy(b).cuda(),
                   w_is_nk)
    r = check_linear(y.double().cpu().numpy(), x.astype(np.float64), w.astype(np.float64),
                     None if b is None else b.astype(np.float64), w_is_nk)
    print(f"jk_f32_linear M {M} N {N} K {K} w_is_nk {w_is_nk} bias {bias}: err / gamma bound {r:.3e}")


def test_f32_linear_upsampler_size():
    # the x_out product of 16 samples of the bottom upsampler's whole window (2048 x 1920), 40 rows more so that the last
    # 64-row tile is partial; float64 on a sample of rows, the whole last tile included
    M, N, K = 16 * 8192 + 40, 2048, 1920
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) * 0.02
    y = f32_linear(x, w, None, 1)
    rng = np.random.RandomState(7)
    rows = np.unique(np.concatenate([[0], rng.randint(0, M, 64), np.arange(M - 40 - 24, M)]))
    ri = torch.from_numpy(rows).cuda()
    r = check_linear(y[ri].double().cpu().numpy(), x[ri].double().cpu().numpy(), w.double().cpu().numpy(), None, 1)
    print(f"jk_f32_linear M {M} N {N} K {K}: {len(rows)} rows, err / gamma bound {r:.3e}")
