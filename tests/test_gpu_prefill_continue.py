"""Continuation prefill: jk_prior_prefill on an engine at position t0 > 0 runs positions t0 .. t0+P-1 on top of the rows'
K / V caches, with the new queries attending from the cache (csrc/prefill.cu).

1. The attention kernels on their own (jk_prefill_attention_f16 with q_offset / cache_rows / blocks) against float64 at
   the 64-query / 32-key tile edges, on the tensor-core routes (16-byte and 4-byte staging, dh 150) and the scalar
   kernels, with the bounds of test_gpu_prefill_attn.py.  The cache holds the keys of positions [0, t0 + P) as the
   engine leaves them (each position written to its decode row in order, so a ring keeps the last writers); the rows
   nothing wrote and the K / V columns of qkv (a continuation reads its keys from the cache only) are NaN.
2. The engine: for every attn_func, the outputs of a continuation and the logits of the steps after it against one
   prefill of [0, t0 + P) and against stepping, with the bounds test_gpu_prefill.py uses (3e-3 for logits, 5e-3 for the
   stack's output; against stepping, no farther than the one prefill is from it, whose own distance is that floor on
   the 16-layer stack); chains of three calls; rows after a select fan-out; every error case, which must leave the
   position where it was."""
import ctypes as C
import zlib
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from golden_util import rel_err
from jukebox_b200 import _lib
from jukebox_b200._lib import lib, stream_ptr
from test_gpu_prefill_attn import GUARD, exact_grid, key_lists, key_mask, nan16, reference, with_guard

pytestmark = pytest.mark.gpu

TOL = 3e-3          # test_gpu_prefill.py: logits, prefill vs stepping
TOL_H = 5e-3        # test_gpu_prefill.py (only_encode): the stack's output h, prefill vs stepping


# ---- 1. the kernels against float64 ----------------------------------------------------------------------------------
def cache_row(f, p, bc, blocks):
    """decode_engine.cu attn_geom.wrow of position p"""
    return {0: p, 1: p % bc if bc else 0, 2: (p % bc) * blocks + p // bc if bc else 0,
            3: ((p // bc) & 1) * bc + p % bc if bc else 0, 7: p}[f]


@dataclass
class Cont:
    name: str
    attn_func: int
    dh: int
    t0: int
    P: int
    n: int = 1
    H: int = 2
    bc: int = 0
    blocks: int = 0
    prime: int = 0
    enc_rows: int = 0
    route: tuple = None             # (tile_dh, stage_bytes) of route 0; None: the scalar kernels
    exact: bool = True

    @property
    def dh_pad(self):
        return -(-self.dh // 16) * 16

    @property
    def rows(self):
        f = self.attn_func
        return {0: self.t0 + self.P, 1: self.bc, 2: self.bc * self.blocks, 3: 2 * self.bc, 6: self.enc_rows,
                7: self.prime}[f]

    def __str__(self):
        return self.name


R32, R64, R128, R160W4, R256W4 = (32, 16), (64, 16), (128, 16), (160, 4), (256, 4)
CONT = [
    *[Cont(f"dh64-dense-t{t0}-P{P}", 0, 64, t0, P, n=2, route=R64)
      for t0, P in ((1, 1), (1, 63), (31, 1), (31, 34), (32, 64), (33, 65), (63, 2), (64, 130), (200, 129))],
    Cont("dh16-dense-t95-P33", 0, 16, 95, 33, n=2, H=3, route=R32),
    Cont("dh128-dense-t1000-P64", 0, 128, 1000, 64, route=R128),
    Cont("dh64-block-bc128-t129-P63", 1, 64, 129, 63, bc=128, route=R64),
    Cont("dh64-block-bc128-t192-P64", 1, 64, 192, 64, bc=128, route=R64),
    Cont("dh64-block-bc16-t17-P1", 1, 64, 17, 1, n=3, bc=16, route=R64),
    Cont("dh64-transpose-bc16-t1000-P100", 2, 64, 1000, 100, bc=16, blocks=80, route=R64),
    Cont("dh64-transpose-bc16-t15-P3", 2, 64, 15, 3, n=2, bc=16, blocks=4, route=R64),
    Cont("dh64-prevblock-bc65-t133-P120", 3, 64, 133, 120, n=2, bc=65, route=R64),
    Cont("dh64-prevblock-bc32-t1-P31", 3, 64, 1, 31, bc=32, route=R64),
    Cont("dh64-prevblock-bc32-t31-P33", 3, 64, 31, 33, bc=32, route=R64),
    *[Cont(f"dh64-prime48-t{t0}-P{P}", 7, 64, t0, P, prime=48, route=R64) for t0, P in ((30, 40), (47, 2), (60, 10))],
    Cont("dh128-encdec-rows33-t50-P70", 6, 128, 50, 70, n=2, enc_rows=33, route=R128),
    Cont("dh150-dense-t77-P65", 0, 150, 77, 65, route=R160W4),
    Cont("dh150-transpose-bc128-t1000-P300", 2, 150, 1000, 300, bc=128, blocks=16, route=R160W4),
    Cont("dh150-block-bc128-t130-P100", 1, 150, 130, 100, bc=128, route=R160W4),
    Cont("dh150-prevblock-bc128-t200-P150", 3, 150, 200, 150, bc=128, route=R160W4),
    Cont("dh150-encdec-rows512-t9-P40", 6, 150, 9, 40, enc_rows=512, route=R160W4),
    Cont("dh170-dense-t70-P40", 0, 170, 70, 40, route=R256W4),
    Cont("dh480-block-bc128-t140-P100", 1, 480, 140, 100, bc=128),
    Cont("dh75-transpose-bc8-t60-P30", 2, 75, 60, 30, bc=8, blocks=16),
    Cont("real-dh64-dense-t500-P100", 0, 64, 500, 100, route=R64, exact=False),
    Cont("real-dh150-prevblock-bc128-t300-P200", 3, 150, 300, 200, bc=128, route=R160W4, exact=False),
]


def cont_inputs(c, g):
    """qkv of the new rows (K / V columns NaN), the caches, and the keys by absolute position: q [n, P, H, dh],
    k / v [n, t0+P (or enc_rows), H, dh]"""
    S, T = c.H * c.dh, c.t0 + c.P
    nk = c.enc_rows if c.attn_func == 6 else T

    def qk(shape, lim):
        return exact_grid(shape, lim, g, "cuda") if c.exact else (torch.randn(shape, generator=g, device="cuda") * 1.5).half()

    rq = torch.randint(1, 25, (c.n, c.P, c.H, 1), generator=g, device="cuda")
    q = qk((c.n, c.P, c.H, c.dh), rq)
    k = qk((c.n, nk, c.H, c.dh), 8)
    v = torch.randn((c.n, nk, c.H, c.dh), generator=g, device="cuda").half()
    kc, vc = nan16((c.n, c.H, c.rows, c.dh_pad)), nan16((c.n, c.H, c.rows, c.dh_pad))
    if c.attn_func == 6:
        kc[..., :c.dh], vc[..., :c.dh] = k.permute(0, 2, 1, 3), v.permute(0, 2, 1, 3)
        return q.reshape(c.n * c.P, S).contiguous(), kc, vc, q, k, v
    # the engine's writes in position order; a previous-block ring is read one block behind, so it holds the blocks
    # before the last one the queries touch
    upto = T if c.attn_func != 3 else (T - 1) // c.bc * c.bc
    for p in range(upto):
        if c.attn_func == 7 and p >= c.prime:
            break
        r = cache_row(c.attn_func, p, c.bc, c.blocks)
        kc[:, :, r, :c.dh], vc[:, :, r, :c.dh] = k[:, p], v[:, p]
    qkv = torch.cat([q.reshape(c.n, c.P, S), nan16((c.n, c.P, 2 * S))], 2)
    return qkv.reshape(c.n * c.P, 3 * S).contiguous(), kc, vc, q, k, v


def run_cont(c, route):
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.name.encode()))
    qkv, kc, vc, q, k, v = cont_inputs(c, g)
    out, out_guard = with_guard(c.n * c.P * c.H * c.dh, g)
    a = _lib.PrefillAttnArgs(qkv=qkv.data_ptr(), k_cache=kc.data_ptr(), v_cache=vc.data_ptr(), out=out.data_ptr(), w=None,
                             ld=0, n=c.n, P=c.P, heads=c.H, dh=c.dh, dh_pad=c.dh_pad, attn_func=c.attn_func, bc=c.bc,
                             prime=c.prime, enc_rows=c.enc_rows, route=route, q_offset=c.t0,
                             cache_rows=0 if c.attn_func == 6 else c.rows, blocks=c.blocks)
    taken = _lib.PrefillAttnRoute()
    rc = lib().jk_prefill_attention_f16(C.byref(a), C.byref(taken), stream_ptr())
    assert rc == 0, lib().jk_last_error().decode()
    torch.cuda.synchronize()
    want = (1, *c.route) if route == 0 and c.route else (0, 0, 0)
    assert (taken.tensor_cores, taken.tile_dh, taken.stage_bytes) == want
    assert torch.equal(out[-GUARD:], out_guard), f"{c}: store past the end of out"
    return out[:-GUARD].view(c.n, c.P, c.H, c.dh), q, k, v


@pytest.mark.parametrize("route", [0, 1])
@pytest.mark.parametrize("case", CONT, ids=str)
def test_continuation_attention_against_float64(case, route):
    c = case
    out, q, k, v = run_cont(c, route)
    T = c.t0 + c.P
    mask = key_mask(c.attn_func, T, c.bc, c.prime, c.enc_rows, "cuda")[c.t0:]     # the new queries' rows
    idx, valid = key_lists(mask)
    no_keys = ~mask.any(1)
    worst = 0.0
    for b in range(c.n):
        for h in range(c.H):
            o_ref, o_bnd, _, _ = reference(q[b, :, h], k[b, :, h], v[b, :, h], idx, valid, c.dh, c.exact)
            o = out[b, :, h].double()
            assert not torch.isnan(o).any(), f"{c} b{b} h{h}: NaN in the output (unwritten, or a poisoned read)"
            assert (o[no_keys] == 0).all(), f"{c} b{b} h{h}: a row without keys is not 0"
            err = (o - o_ref).abs()
            bad = err > o_bnd
            if bad.any():
                p, d = [int(t) for t in bad.nonzero()[0]]
                pytest.fail(f"{c} route {route} b{b} h{h}: {int(bad.sum())} elements out of bound, first position "
                            f"{c.t0 + p} d {d}: {o[p, d].item()} vs {o_ref[p, d].item()} (bound {o_bnd[p, d].item():.3g})")
            worst = max(worst, float((err / o_bnd.clamp_min(1e-30)).max()))
    print(f"{c} route {route}: worst output error {worst:.3f} of its bound")


def test_continuation_attention_rejects_bad_arguments():
    c = Cont("x", 0, 64, 10, 8)
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv, kc, vc, *_ = cont_inputs(c, g)
    out = nan16((c.P, c.H * c.dh))
    base = dict(qkv=qkv.data_ptr(), k_cache=kc.data_ptr(), v_cache=vc.data_ptr(), out=out.data_ptr(), ld=0, n=1, P=c.P,
                heads=c.H, dh=c.dh, dh_pad=c.dh_pad, attn_func=0, q_offset=10, cache_rows=18)
    for bad in (dict(cache_rows=17), dict(q_offset=-1), dict(k_cache=None), dict(attn_func=2, bc=4, blocks=4),
                dict(w=out.data_ptr(), ld=4)):
        a = _lib.PrefillAttnArgs(**{**base, **bad})
        assert lib().jk_prefill_attention_f16(C.byref(a), None, stream_ptr()) != 0, bad
    torch.cuda.synchronize()
    assert torch.isnan(out).all(), "a rejected call wrote its output"


# ---- 2. the engine -----------------------------------------------------------------------------------------------------
def _prior(order, width, depth, heads, n_ctx, blocks, prime_len=None, encoder_dims=0, seed=0, x_cond=False):
    from test_gpu_prefill import _model
    if not encoder_dims:
        return _model(order, width, depth, heads, n_ctx, blocks, prime_len, seed=seed, x_cond=x_cond)[0]
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    from oracle.synth import synth_state_dict
    m = ConditionalAutoregressive2D((n_ctx,), 64, width=width, depth=depth, heads=heads, attn_order=order, blocks=blocks,
                                    x_cond=x_cond, y_cond=True, encoder_dims=encoder_dims)
    sd = m.state_dict()
    w = synth_state_dict([(k, tuple(v.shape)) for k, v in sd.items() if k != "x_out.weight"], seed)
    w["x_out.weight"] = w["x_emb.weight"]
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()}, strict=True)
    return m.cuda().eval()


# attn_order 12: block / transpose / previous block / prime layers (the single_enc_dec stack); 2: block / transpose /
# previous block (upsampler-like); 0: dense; 6: with encoder-decoder layers (the sep_enc_dec decoder)
STACKS = {
    "order12": dict(order=12, width=256, depth=16, heads=2, n_ctx=96, blocks=8, prime_len=24),
    "order2": dict(order=2, width=256, depth=6, heads=1, n_ctx=64, blocks=4),
    "dense": dict(order=0, width=256, depth=3, heads=4, n_ctx=48, blocks=None),
    "encdec": dict(order=6, width=256, depth=8, heads=2, n_ctx=64, blocks=4, encoder_dims=24, x_cond=True),
    "dh150": dict(order=2, width=4800, depth=3, heads=8, n_ctx=64, blocks=4),
}


class Setup:
    def __init__(self, key, n=5, seed=0):
        kw = dict(STACKS[key])
        self.m = m = _prior(**kw, seed=seed)
        self.n_ctx, self.n = kw["n_ctx"], n
        self.bc = kw["n_ctx"] // kw["blocks"] if kw.get("blocks") else kw["n_ctx"]
        g = torch.Generator().manual_seed(seed + 17)
        self.tokens = torch.randint(0, m.bins, (n, self.n_ctx), generator=g).cuda()
        self.yc = torch.randn(n, m.width, generator=g).cuda()
        self.xc = (0.1 * torch.randn(n, self.n_ctx, m.width, generator=g)).cuda() if kw.get("x_cond") else None
        self.ekv = torch.randn(n, kw["encoder_dims"], m.width, generator=g).cuda() if kw.get("encoder_dims") else None

    def engine(self):
        m = self.m
        m.transformer.del_cache()
        eng = m._fresh_engine(self.n, self.ekv)
        eng.reset(0)
        return eng

    def run(self, plan, K):
        """plan: a list of ("step", count) / ("prefill", count); returns (h of every position the plan ran [n, T, W],
        logits of K steps after it [n, K, bins])"""
        m, n = self.m, self.n
        eng = self.engine()
        hs = []
        for how, cnt in plan:
            if how == "prefill":
                h = torch.empty(n, cnt, m.width, device="cuda")
                t0 = eng.position
                eng.prefill(n, cnt, tokens=self.tokens, y_cond=self.yc, x_cond=self.xc, h_out=h)
                assert eng.position == t0 + cnt
                hs.append(h)
            else:
                for _ in range(cnt):
                    o = torch.empty(n, m.width, device="cuda")
                    eng.step(n, tokens=self.tokens, y_cond=self.yc, x_cond=self.xc, h_out=o)
                    hs.append(o[:, None])
        lbuf = torch.empty(n, m.bins, device="cuda")
        out = torch.empty(n, K, m.bins, device="cuda")
        for k in range(K):
            eng.step(n, tokens=self.tokens, y_cond=self.yc, x_cond=self.xc, logits=lbuf)
            out[:, k] = lbuf
        torch.cuda.synchronize()
        m.transformer.del_cache()
        return torch.cat(hs, 1).cpu().numpy(), out.cpu().numpy()


def _t0s(n_ctx, bc):
    return sorted({1, bc - 1, bc, bc + 1, 2 * bc + 3, n_ctx - 2})


def _chunks(t0, n_ctx, bc):
    """chunk lengths from t0: crossing no block edge (if there is room), one, several, and ending at n_ctx"""
    to_edge = (t0 // bc + 1) * bc - t0
    out = {1, n_ctx - t0}
    if to_edge > 1:
        out.add(to_edge - 1)
    out.add(min(n_ctx - t0, to_edge + 1))
    out.add(min(n_ctx - t0, to_edge + 2 * bc + 1))
    return sorted(p for p in out if 1 <= p <= n_ctx - t0)


@pytest.mark.parametrize("key", list(STACKS))
def test_continuation_matches_one_prefill_and_stepping(key):
    s = Setup(key, seed=len(key))
    K, worst = 6, 0.0          # test_gpu_prefill.py: 5 rows, the logits of 6 steps
    for t0 in _t0s(s.n_ctx, s.bc):
        for P in _chunks(t0, s.n_ctx, s.bc):
            k = min(K, s.n_ctx - t0 - P)
            ha, la = s.run([("prefill", t0), ("prefill", P)], k)
            hb, lb = s.run([("prefill", t0 + P)], k)
            hc, lc = s.run([("step", t0 + P)], k)
            eh = max(rel_err(ha[:, t0:], hb[:, t0:]), rel_err(ha[:, t0:], hc[:, t0:]))
            assert np.isfinite(ha).all() and np.isfinite(la).all()
            assert eh < TOL_H, f"{key} t0 {t0} P {P}: h of the continuation vs one prefill / stepping {eh:.2e}"
            if k:
                # against one prefill: within TOL.  Against stepping: the prefill's own distance from stepping is the
                # fp32 summation-order floor, at TOL on the 16-layer stack; the continuation must be no farther
                e_cp, e_cs, e_ps = rel_err(la, lb), rel_err(la, lc), rel_err(lb, lc)
                assert e_cp < TOL and e_cs < max(TOL, e_ps + TOL / 10), \
                    f"{key} t0 {t0} P {P}: logits of the continuation vs one prefill {e_cp:.2e}, vs stepping {e_cs:.2e} " \
                    f"(one prefill vs stepping {e_ps:.2e})"
                worst = max(worst, e_cp, e_cs)
    print(f"{key}: worst continuation logits error {worst:.2e}")


@pytest.mark.parametrize("key", ["order12", "encdec"])
def test_three_chained_continuations(key):
    s = Setup(key, seed=5)
    bc, T = s.bc, s.n_ctx
    for cuts in ((5, bc + 2, 2 * bc + 1), (bc, bc, T - 2 * bc - 3), (1, 1, T - 4)):
        plan = [("step", 2)] + [("prefill", c) for c in cuts]
        used = 2 + sum(cuts)
        k = min(2, T - used)
        ha, la = s.run(plan, k)
        hb, lb = s.run([("step", used)], k)
        eh, el = rel_err(ha, hb), (rel_err(la, lb) if k else 0.0)
        assert eh < TOL_H and el < TOL, f"{key} chain {cuts}: h {eh:.2e}, logits {el:.2e}"


def test_rows_follow_their_own_histories_after_a_fan_out():
    """a prime on one row, fanned out to 4 rows (select), then each row's own tokens continued by one prefill: every
    row's logits match a fresh run of that row's whole history"""
    s = Setup("order12", n=4, seed=9)
    m, n, prime, P = s.m, 4, 30, 40
    tok = s.tokens.clone()
    tok[:, :prime] = tok[:1, :prime]
    yc = s.yc[:1].expand(n, -1).contiguous()
    eng = s.engine()
    eng.prefill(1, prime, tokens=tok[:1], y_cond=yc[:1])
    eng.select([0] * n)
    h = torch.empty(n, P, m.width, device="cuda")
    eng.prefill(n, P, tokens=tok, y_cond=yc, h_out=h)
    lbuf = torch.empty(n, m.bins, device="cuda")
    eng.step(n, tokens=tok, y_cond=yc, logits=lbuf)
    got = lbuf.cpu().numpy()
    m.transformer.del_cache()
    s.tokens, s.yc = tok, yc
    hr, lr = s.run([("step", prime + P)], 1)
    assert rel_err(h.cpu().numpy(), hr[:, prime:]) < TOL_H
    assert rel_err(got, lr[:, 0]) < TOL


def test_continuation_errors_leave_the_position():
    s = Setup("order12", seed=3)
    m, n, T = s.m, s.n, s.n_ctx
    eng = s.engine()
    eng.prefill(n, 10, tokens=s.tokens, y_cond=s.yc)
    cap = eng.prefill_capacity
    w = torch.zeros(n, m.transformer.n_head, 4, 4, dtype=torch.float16, device="cuda")
    from jukebox_b200.engine import Capture
    cases = [dict(n_positions=T - 10 + 1), dict(n_positions=cap + 1), dict(n_positions=4, record={0: w}),
             dict(n_positions=4, n_layers=1),
             dict(n_positions=4, capture={0: Capture(torch.empty(n, m.width, device="cuda"), 0, 4, True, False)})]
    for kw in cases:
        P = kw.pop("n_positions")
        with pytest.raises(RuntimeError):
            eng.prefill(n, P, tokens=s.tokens, **kw)
        assert eng.position == 10
        t = C.c_int(-5)
        _lib.check(lib().jk_prior_position(eng.handle, C.byref(t)))
        assert t.value == 10, f"{kw}: the position moved to {t.value}"
    # a truncated engine (position -1) refuses a continuation as it refuses a step
    eng.reset(0)
    eng.prefill(n, 10, tokens=s.tokens, y_cond=s.yc, n_layers=1)
    with pytest.raises(RuntimeError):
        eng.prefill(n, 4, tokens=s.tokens)
    m.transformer.del_cache()
