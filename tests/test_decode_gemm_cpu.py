"""The Conv1D partition restated in oracle/decode_gemm.py, its bound, and the GPU file's checks against planted faults
(no GPU: jk_prior_plan is host arithmetic, the rest numpy).

Dealing: for every configuration of test_decode_plan_cpu.CONFIGS on 132 and 114 SMs, with the 16- and 32-row layouts
(the ring differs, so the in_order phases differ), every k-step of every (CTA, Conv1D, layer) goes to exactly one warp,
nwarp counts exactly the warps that multiplied, and the epilogue writes every (row, column pair) once.
Bound: the emulation of the kernel's order, with a round-to-nearest MMA and with the truncating model, stays within
decode_gemm.bound, also on rows whose sums cancel; the largest err / bound is printed.
Planted faults: each emulation with one fault fails the GPU file's exact check (and its rounding check) at the probe
shapes; a Q-unit k-step dropped fails the attention check of part c."""
import json

import numpy as np
import pytest

from oracle import decode_attn as da
from oracle import decode_gemm as dg
from oracle.decode_stats import staged
from test_decode_plan_cpu import CONFIGS, plan


def record(row):
    print(json.dumps(row))


def plan_at(name, sms, mb):
    w = CONFIGS[name]
    CONFIGS[name] = w[:9] + (mb,) + w[10:]
    try:
        return plan(name, sms)
    finally:
        CONFIGS[name] = w


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("rows", [16, 32])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_every_kstep_dealt_once(name, rows, sms):
    try:
        cfg, info, cols = plan_at(name, sms, rows)
    except RuntimeError as e:
        assert rows == 32 and "takes at most 16 samples" in str(e)      # 5b_lyrics: the 32-row tile does not fit
        pytest.skip(f"{name} has no {rows}-row layout")
    Ks = [cfg.width, cfg.n_state, cfg.width, cfg.mlp_width]
    seen = set()
    for l in range(cfg.depth):
        for gi in range(4):
            for ncg in set(int(n) for n in cols[:, l, gi, 1]):
                if ncg == 0 or (gi, ncg) in seen:
                    continue
                seen.add((gi, ncg))
                ph = dg.Phase(Ks[gi], info.k_split, ncg, info.ring_slots)
                dealt = [k for w in ph.steps for k in w]
                assert sorted(dealt) == list(range(ph.nkk)), (name, gi, ncg)
                assert [w for w in range(8) if ph.steps[w]] == list(range(ph.nwarp)), (name, gi, ncg)
                for w in ph.steps:
                    assert w == sorted(w)
                fin = ph.finished(rows)
                got = sorted((b, p) for _, _, _, b, p in fin)
                assert got == [(b, p) for b in range(rows) for p in range(4 * ncg)], (name, gi, ncg)


def _operands(rng, B, K, N, mode):
    """probe-shaped operands: staged LayerNorm rows and grid weights (exact), or real LayerNorm rows and dense
    weights (rounding)"""
    if mode == "exact":
        g, b = dg.exact_ln(rng, K)
        x = dg.grid_rows(rng, B, K).astype(np.float16)
        return staged(x, g, b), dg.weights16(dg.grid_weights(rng, K, N)), dg.bias32(dg.grid_bias(rng, N))
    x = rng.standard_normal((B, K)).astype(np.float16)
    g = (1 + 0.1 * rng.standard_normal(K)).astype(np.float32)
    b = (0.1 * rng.standard_normal(K)).astype(np.float32)
    w = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    return staged(x, g, b), dg.weights16(w), dg.bias32(0.1 * rng.standard_normal(N))


# (K, KS, ncg, ring slots): 1b QKV, 5b fc (in_order), small_upsampler proj (nkk 4 < 8 warps), 1104 QKV (KS 1, ncg 1),
# 5b proj (one-row epilogue layout, in_order)
PHASES = {"1b_qkv": (2048, 4, 8, 5), "5b_fc": (4800, 1, 4, 3), "small_up_proj": (256, 4, 4, 5),
          "1104_qkv": (1104, 1, 1, 7), "5b_proj": (1200, 1, 5, 3)}


@pytest.mark.parametrize("which", list(PHASES))
def test_emulation_within_bound(which):
    K, KS, ncg, slots = PHASES[which]
    ph = dg.Phase(K, KS, ncg, slots)
    rng = np.random.default_rng(1)
    N = 8 * ncg
    worst = {}
    for rows in ("random", "cancelling"):
        A, W, b = _operands(rng, 32, K, N, "round")
        if rows == "cancelling":
            # half the products of each column cancel the other half up to a few ulps: the result is tiny against
            # sum |a w|, where a relative error bound would be smallest and the absolute one matters
            A = A.copy()
            h = K // 2
            A[:, h:2 * h] = -A[:, :h]
            W = W.copy()
            W[h:2 * h] = W[:h]
            W[h + rng.integers(0, h, 4)] *= np.float16(1.001)
        sb, bd = dg.bound(A, W, b, ph)
        for mma in ("rn", "trunc"):
            y = dg.emulate(A, W, b, ph, mma=mma)
            # the fp32 value before the fp16 rounding lies within the bound: its fp16 rounding is admissible
            y64 = y.astype(np.float64)
            assert ((dg.f16(sb - bd) <= y64) & (y64 <= dg.f16(sb + bd))).all(), (which, rows, mma)
            y32 = _emulate32(A, W, b, ph, mma)
            r = float((np.abs(y32 - sb) / bd).max())
            assert r <= 1.0, (which, rows, mma, r)
            worst[f"{rows}/{mma}"] = round(r, 4)
    record(dict(case="emulation vs bound", phase=which, K=K, KS=KS, ncg=ncg, in_order=ph.in_order, nwarp=ph.nwarp,
                max_err_over_bound=worst))


def _emulate32(A, W, b, ph, mma):
    """the fp32 value fl(s + b) before the fp16 rounding, by the emulation's order"""
    f = dg._mma_rn if mma == "rn" else dg._mma_trunc
    A64, W64 = np.asarray(A, np.float64), np.asarray(W, np.float64)
    s = np.zeros((A.shape[0], W.shape[1]), np.float32)
    for r in range(ph.KS):
        t = np.zeros_like(s)
        for w in range(ph.nwarp):
            C = np.zeros_like(s)
            for kk in ph.steps[w]:
                sl = slice(r * ph.Ks + 16 * kk, r * ph.Ks + 16 * kk + 16)
                C = f(C, A64[:, sl], W64[sl])
            t = (t + C).astype(np.float32)
        s = (s + t).astype(np.float32)
    return (s + np.asarray(b, np.float32)).astype(np.float32).astype(np.float64)


# planted fault: (phase, mutation of Phase or of emulate)
FAULTS = {"in_order k-step dropped": ("5b_fc", "in_order_drop", None),
          "in_order k-step dealt twice": ("5b_fc", "in_order_twice", None),
          "rank partial missing": ("1b_qkv", None, "rank_missing"),
          "rank partial from the previous Conv1D": ("1b_qkv", None, "rank_stale"),
          "pr = pl (rank offset lost)": ("1b_qkv", None, "pair_no_rank_offset"),
          "bias of the neighbouring pair": ("1b_qkv", None, "bias_next_pair"),
          "rows 16-31 from the first m16 tile": ("1b_qkv", None, "rows_tile0")}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_planted_fault_fails_the_checks(fault):
    which, ph_mut, emu_mut = FAULTS[fault]
    K, KS, ncg, slots = PHASES[which]
    rng = np.random.default_rng(2)
    N = 3 * 8 * ncg                                    # three units of this ncg
    out = {}
    for mode in ("exact", "round"):
        A, W, b = _operands(rng, 32, K, N, mode)
        ph = dg.Phase(K, KS, ncg, slots)
        other = rng.standard_normal((32, N)).astype(np.float32) if emu_mut == "rank_stale" else None
        y = dg.emulate(A, W, b, dg.Phase(K, KS, ncg, slots, mutate=ph_mut), mutate=emu_mut, other=other)
        if mode == "exact":
            assert dg.exact_in_fp32(A, W, b)
            sb, bd = dg.conv64(A, W, b), np.zeros((32, N))
        else:
            sb, bd = dg.bound(A, W, b, ph)
        lo, hi, _, _ = dg.admissible("qkv", sb, bd)
        assert dg.in_interval(dg.emulate(A, W, b, ph), lo, hi).all()          # the fault-free kernel passes
        ok = dg.in_interval(y, lo, hi)
        out[mode] = int((~ok).sum())
        assert (~ok).any(), (fault, mode)
    record(dict(case="planted fault", fault=fault, phase=which, elements_failing=out))


def test_planted_q_fault_fails_the_attention_check():
    """a k-step of one Q unit dropped: q moves, and the attention output of part c leaves decode_attn.bound"""
    rng = np.random.default_rng(3)
    W, S, H = 2048, 512, 2
    dh = S // H
    g = da.Geom(heads=H, dh=dh, n_ctx=16, blocks=4, G=132)
    gamma, beta = dg.exact_ln(rng, W)
    wq = dg.weights16(dg.grid_weights(rng, W, S))
    wk = dg.weights16(dg.grid_weights(rng, W, S))
    Av = rng.permutation(W)[:S]
    pos = 3                                            # keys of 3 positions (pattern 2 at p = 11: rows 3, 7, 11)
    rows = staged(dg.grid_rows(rng, pos, W).astype(np.float16), gamma, beta)
    K = dg.f16(dg.conv64(rows, wk))
    V = rows[:, Av]
    q = dg.f16(dg.conv64(rows[-1:], wq))[0]
    wq_bad = wq.copy()
    wq_bad[16 * 5:16 * 6, 0:64] = 0                    # k-step 5 lost for the columns of one unit (8 groups)
    q_bad = dg.f16(dg.conv64(rows[-1:], wq_bad))[0]
    parts = da.partition(g, pos - 1, 1, 1)
    fails, worst = 0, 0.0
    for h in range(H):
        sl = slice(h * dh, (h + 1) * dh)
        bd, a, _ = da.bound(q[sl], K[:, sl], V[:, sl], g, parts)
        _, _, a_bad = da.attend64(q_bad[sl], K[:, sl], V[:, sl], g.scale2)
        ok = np.abs(a_bad - a) <= bd
        fails += int((~ok).sum())
        worst = max(worst, float((np.abs(a_bad - a) / bd).max()))
    record(dict(case="planted fault", fault="Q-unit k-step dropped", elements_failing=fails, max_err_over_bound=worst))
    assert fails > 0
