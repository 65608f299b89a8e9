"""The decode step's attention (csrc/decode_engine.cu attn_item) against float64 at the priors' real geometry, through
every pattern, split and tile edge.

A probe layer makes attention the only inexact stage.  The W columns split into four disjoint sets of S = W / 4: A_q,
A_k, A_v and B (a fixed random permutation).  Input rows are zero on B; LN0 has gamma = 1, beta = 0; c_attn selects
q_j = 2^e LN0(x)[A_q[j]], k_j = LN0(x)[A_k[j]], v_j = LN0(x)[A_v[j]] (one nonzero product per output: exact fp16 values
that numpy gets from oracle/decode_stats.staged); c_proj puts attention dim j back into column B[j]; the MLP is zero.
So h_out[:, B] is the kernel's fp16 attention output and h_out equals x elsewhere; both are asserted.  For the
encoder-decoder layer c_attn holds q alone and c_enc_kv selects the encoder's A_k / A_v columns, so K / V = fp16(enc).

Rows: every row is a rotation of one of 256 base rows on A_q + A_k + A_v (i -> i + c mod 3S), no (base, c) twice in a
run, so no two positions share a key.  The fixed-point LayerNorm statistics do not depend on the order of a row, so LN0
of a row is its base row's LN0, rotated: numpy knows every cached k / v without a LayerNorm per position.

Caches are filled by stepping from position 0.  At probe positions (chosen from the restated partition in
oracle/decode_attn.py: every split transition, ncache at k (RC-1) and k (RC-1) + 1, a full last tile, nr = 0 and 1 mod
16, block edges, the prime edge, the last position) the engine is rewound to the probe (reset(p) keeps the caches) and:
  * bounded numerics: for e in REGIMES every (sample, head, dim) is within oracle/decode_attn.bound of the float64
    attention (near-uniform over 8576 keys at e = -8, one-hot-like with fp16-subnormal P at e = 3);
  * exact routing: q of position p is built from the key row of one position j* (x_p[A_q] := x_j*[A_k]) with the float64
    score of j* at least 40 above every other and sum_{j != j*} e^{s_j - s*} max|v| < 2^-26; wherever both hold (all but
    a few (sample, head) pairs whose key has a small norm, at most 1 in 20, asserted) the kernel must return v_j* bit
    for bit.  j* sits at the first and last row of a tile and of parts 0 and ns - 1, the current
    token, both ends of every ring, the last prime row and encoder rows 0 and 511;
  * negative routing: j* where the pattern must not look (the previous block for pattern 1, the current block for 3, the
    current token and rows past the padded prime for 7, another sample, another head): the output is the oracle's
    (within the bound) and not v_j*;
then the position is stepped once more with its own row, which leaves the caches as the fill made them.

One JSON line per probe (pytest -s); test_coverage restates what the cases' probes visit and asserts it."""
import ctypes as C
import json
import math
import time
from collections import defaultdict
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from jukebox_b200 import _lib
from jukebox_b200.engine import DecodeEngine, prior_config
from oracle import decode_attn as da
from oracle.decode_stats import staged
from test_gpu_decode_geometry import to_cuda, zero_block

pytestmark = pytest.mark.gpu

# width, heads, n_ctx, blocks, prime_len, encoder rows, max batch (the full-size fixtures' configurations, and a width
# with 16 heads of 32 dims, so that B * H passes the SM count and CTAs take items that were not prefetched)
GEOM = {"1b": (2048, 2, 8576, 64, 384, 0, 32),
        "5b": (4800, 8, 8192, 128, 0, 512, 16),
        "up": (1920, 1, 8192, 128, 0, 0, 32),
        "many": (2048, 16, 1024, 16, 0, 0, 32)}
CASES = [(0, "1b"), (1, "1b"), (1, "5b"), (1, "up"), (2, "1b"), (2, "5b"), (2, "up"),
         (3, "1b"), (3, "5b"), (3, "up"), (6, "5b"), (7, "1b"), (0, "many")]
REGIMES = (-8, -2, 0, 2, 3)
N_BASE = 256


def record(row):
    print(json.dumps(row))


def sm_count():
    out = C.c_int(0)
    _lib.check(_lib.lib().jk_device_sm_count(C.byref(out)))
    return out.value


def tile_rows(cfg, G):
    info = _lib.PlanInfo()
    _lib.check(_lib.lib().jk_prior_plan(C.byref(cfg), G, C.byref(info), None, 0))
    return info.tile_rows


def batches(g, af, maxb):
    """per distinct (largest split the pattern reaches, 16- or 32-row kernel): the largest batch that gives it"""
    max_ncache = {0: g.n_ctx - 1, 1: g.bc - 1, 2: g.blocks - 1, 3: g.bc, 6: g.enc_dims, 7: g.prime_pad}[af]
    ns_cap = da.attn_nsplit(g, 4, max_ncache)
    seen = {}
    for B in range(maxb, 0, -1):
        key = (min(da.gmax_of(g, B), ns_cap), B > 16)
        seen.setdefault(key, B)
    return sorted(seen.values())


def route_exponent(dh):
    """2^e for the routing query: the aligned score grows as 2^e 1.33 sqrt(dh), the others as about 2^e 1.33 4.5, and
    |k|^2 spreads more at small head dims (two more octaves below 64 dims); q . k stays far below the fp16 maximum"""
    e = math.ceil(math.log2(80 / (1.33 * (math.sqrt(dh) - 4.5)))) + (2 if dh < 64 else 0)
    return int(min(8, max(1, e)))


def probe_positions(g, af, B, t_end):
    """the first position of every feature of the restated partition, and the last position"""
    gm = da.gmax_of(g, B)
    chosen, prev_ns = {}, None
    for p in range(t_end):
        R, _, cur, _ = da.attn_geom(g, af, p)
        tags = []
        if R == 0:
            ns = 0
            tags.append("zeros")
        else:
            nc = da.ncache_of(R, cur)
            ns = da.attn_nsplit(g, gm, nc)
            parts = da.partition(g, nc, ns, cur)
            _, nr, withcur = parts[-1]["tiles"][-1]
            nr += withcur
            tags += [("ns", ns), ("ntiles", min(3, max(len(pt["tiles"]) for pt in parts)))]
            if prev_ns is not None and ns != prev_ns:
                tags.append(("ns_change", prev_ns, ns))
            if nc and nc % g.trows in (0, 1):
                tags.append(("ncache mod RC-1", nc % g.trows, min(nc // g.trows, 5)))
            if nr == g.RC:
                tags.append("full last tile")
            if nr % 16 in (0, 1):
                tags.append(("nr mod 16", nr % 16))
        if af != 6 and p % g.bc in (0, g.bc - 1):
            tags.append(("block edge", p % g.bc, min(p // g.bc, 2)))
        if af == 7 and p - g.prime_pad in (-1, 0, 1):
            tags.append(("prime edge", p))
        if p == t_end - 1:
            tags.append("last")
        for t in tags:
            chosen.setdefault(t, p)
        prev_ns = ns
    return sorted(set(chosen.values()))


class Probe:
    """a one-layer (or depth-2, layer 0 zero) engine whose last layer is the attention probe, and its numpy model"""

    def __init__(self, af, name, depth=1, seed=0):
        W, H, n_ctx, blocks, prime, enc, maxb = GEOM[name]
        S = W // 4
        self.af, self.name, self.W, self.S, self.H, self.depth, self.maxb = af, name, W, S, H, depth, maxb
        self.eng = DecodeEngine(width=W, depth=depth, heads=H, n_state=S, mlp_width=W, n_ctx=n_ctx, blocks=blocks,
                                attn_funcs=[0] * (depth - 1) + [af], bins=0, prime_len=prime, encoder_dims=enc,
                                max_batch=maxb)
        G = sm_count()
        self.g = da.Geom(heads=H, dh=S // H, n_ctx=n_ctx, blocks=blocks, prime_len=prime, enc_dims=enc, G=G,
                         RC=tile_rows(self.eng.cfg, G))
        assert self.g.RC in [da.attn_tile_rows(self.g.dhp) >> k for k in range(4)]
        rng = np.random.default_rng(1000 + seed)
        perm = rng.permutation(W)
        self.Aq, self.Ak, self.Av, self.Bc = perm[:S], perm[S:2 * S], perm[2 * S:3 * S], perm[3 * S:]
        self.A = perm[:3 * S]
        if depth == 2:
            self.eng.load_layer(0, to_cuda(zero_block(W, S, W)))
        self.blocks = {}

    def block(self, e):
        """the probe layer with q scaled by 2^e (fp16 weights, built once per e)"""
        if e not in self.blocks:
            W, S = self.W, self.S
            blk = zero_block(W, S, W, self.af)
            j = torch.arange(S)
            if self.af == 6:
                blk.attn.c_attn = NS(w=torch.zeros(W, S), b=torch.zeros(S))
                blk.attn.c_enc_kv = NS(w=torch.zeros(W, 2 * S), b=torch.zeros(2 * S))
                blk.attn.c_enc_kv.w[self.Ak, j] = 1.0
                blk.attn.c_enc_kv.w[self.Av, S + j] = 1.0
            else:
                blk.attn.c_attn.w[self.Ak, S + j] = 1.0
                blk.attn.c_attn.w[self.Av, 2 * S + j] = 1.0
            blk.attn.c_attn.w[self.Aq, j] = 2.0 ** e
            blk.attn.c_proj.w[j, self.Bc] = 1.0
            mods = [blk.attn.c_attn, blk.attn.c_proj, blk.mlp.c_fc, blk.mlp.c_proj] + \
                ([blk.attn.c_enc_kv] if self.af == 6 else [])
            for m in mods:
                m.w, m.b = m.w.half(), m.b.half()
            if self.af == 6:
                blk.attn.c_enc_kv = NS(w=blk.attn.c_enc_kv.w.cuda(), b=blk.attn.c_enc_kv.b.cuda())
            self.blocks[e] = to_cuda(blk)
        return self.blocks[e]

    def load(self, e):
        if self.loaded != e:
            self.eng.load_layer(self.depth - 1, self.block(e))
            self.loaded = e

    # ---- rows ------------------------------------------------------------------------------------------------------
    def make_rows(self, B, seed):
        """base rows, their LN0, and per (position, sample) a base row and a permutation; x on the device, k / v / q
        of every position in numpy"""
        W, S, T = self.W, self.S, self.g.n_ctx
        rng = np.random.default_rng(seed)
        # N(0, 1): every row has the same scale, so a query built from another row's values stays aligned with its key
        base = rng.standard_normal((N_BASE, 3 * S)).astype(np.float16)
        full = np.zeros((N_BASE, W), np.float16)
        full[:, self.A] = base
        ln = staged(full, np.ones(W, np.float32), np.zeros(W, np.float32))[:, self.A]
        self.base, self.ln = base, ln
        combo = rng.choice(N_BASE * 3 * S, T * B, replace=False).reshape(T, B)
        self.beta, self.pc = combo // (3 * S), combo % (3 * S)
        self.X = torch.empty(T, B, W, device="cuda")
        base_d = torch.from_numpy(base.astype(np.float32)).cuda()
        self.K = np.empty((B, T, S), np.float16)
        self.V = np.empty((B, T, S), np.float16)
        self.Q = np.empty((B, T, S), np.float16)
        ar = np.arange(3 * S)
        A_d = torch.from_numpy(self.A).cuda()
        for t0 in range(0, T, 256):
            t1 = min(T, t0 + 256)
            idx = (ar + self.pc[t0:t1, :, None]) % (3 * S)                                 # [t, B, 3S]
            rows = self.ln[self.beta[t0:t1, :, None], idx]
            self.Q[:, t0:t1] = rows[..., :S].transpose(1, 0, 2)
            self.K[:, t0:t1] = rows[..., S:2 * S].transpose(1, 0, 2)
            self.V[:, t0:t1] = rows[..., 2 * S:].transpose(1, 0, 2)
            idx_d = torch.from_numpy(idx).cuda()
            vals = base_d[torch.from_numpy(self.beta[t0:t1]).cuda()].gather(2, idx_d)
            x = torch.zeros(t1 - t0, B, W, device="cuda")
            x[:, :, A_d] = vals
            self.X[t0:t1] = x
        if self.af == 6:
            enc = rng.standard_normal((B, self.g.enc_dims, W)).astype(np.float16)
            self.enc = enc
            self.eng.set_encoder_kv(torch.from_numpy(enc.astype(np.float32)).cuda())
            self.KE, self.VE = enc[:, :, self.Ak], enc[:, :, self.Av]

    def x_row(self, t, b):
        x = np.zeros(self.W, np.float16)
        x[self.A] = self.base[self.beta[t, b], (np.arange(3 * self.S) + self.pc[t, b]) % (3 * self.S)]
        return x

    def keys(self, b, pos):
        if self.af == 6:
            return self.KE[b][pos], self.VE[b][pos]
        return self.K[b, pos], self.V[b, pos]

    # ---- one step at position p -------------------------------------------------------------------------------------
    def run(self, p, B, x, e):
        """x [B, W] fp16 rows at position p with q scaled by 2^e: the kernel's attention [B, S] and the model's q / k / v"""
        self.load(e)
        self.eng.reset(p)
        h = torch.full((B, self.W), float("nan"), device="cuda")
        self.eng.step(B, x_in=torch.from_numpy(x.astype(np.float32)).cuda(), h_out=h)
        got = h.cpu().numpy()
        rest = np.setdiff1d(np.arange(self.W), self.Bc)
        stray = int((got[:, rest] != x[:, rest].astype(np.float32)).sum())
        assert stray == 0, f"{stray} columns outside B differ from x"
        ln = staged(x, np.ones(self.W, np.float32), np.zeros(self.W, np.float32))
        q = (ln[:, self.Aq].astype(np.float32) * np.float32(2.0 ** e)).astype(np.float16)
        return got[:, self.Bc], q, ln[:, self.Ak], ln[:, self.Av]


def oracle_heads(pr, B, pos, cur, q, kc, vc, parts, with_bound=True):
    """per (b, h): (bound, a64, K, V) of the query against the attended rows (the current token's k / v from this
    step); without the bound, (None, None, K, V)"""
    g, dh = pr.g, pr.g.dh
    out = []
    for b in range(B):
        K, V = pr.keys(b, pos[:len(pos) - cur])
        if cur:
            K, V = np.vstack([K, kc[b][None]]), np.vstack([V, vc[b][None]])
        row = []
        for h in range(g.H):
            sl = slice(h * dh, (h + 1) * dh)
            bd, a, _ = da.bound(q[b, sl], K[:, sl], V[:, sl], g, parts) if with_bound else (None, None, None)
            row.append((bd, a, K[:, sl], V[:, sl]))
        out.append(row)
    return out


def check_probe(pr, B, p, pos, cur, kind, stats):
    t_start = time.time()
    g, dh, S = pr.g, pr.g.dh, pr.S
    x = pr.X[p].cpu().numpy().astype(np.float16)
    row = dict(geometry=pr.name, pattern=pr.af, B=B, p=p, depth=pr.depth)
    if kind == "zeros":           # pattern 3 inside the first block: keys and values are zeros
        got, *_ = pr.run(p, B, x, 0)
        assert (got == 0).all(), "pattern 3 in the first block must output exactly 0"
        row.update(ns=0, zeros=True)
        record(row)
        return
    nc = len(pos) - cur
    ns = da.attn_nsplit(g, da.gmax_of(g, B), nc)
    parts = da.partition(g, nc, ns, cur)
    its = da.items(g, B, ns, len(pos))
    _, nr, wc = parts[-1]["tiles"][-1]
    row.update(ns=ns, ncache=nc, ntiles=[len(pt["tiles"]) for pt in parts], last_tile_rows=nr + wc,
               prefetched=sum(i["prefetched"] for i in its), not_prefetched=sum(not i["prefetched"] for i in its))
    # bounded numerics
    worst = (0.0, None)
    for e in REGIMES:
        got, q, kc, vc = pr.run(p, B, x, e)
        for b, hs in enumerate(oracle_heads(pr, B, pos, cur, q, kc, vc, parts)):
            for h, (bd, a, _, _) in enumerate(hs):
                r = np.abs(got[b, h * dh:(h + 1) * dh] - a) / bd
                i = int(np.argmax(r))
                if r[i] > worst[0]:
                    worst = (float(r[i]), dict(e=e, b=b, h=h, d=i, err=float(abs(got[b, h * dh + i] - a[i])),
                                               bound=float(bd[i])))
    row.update(max_err_over_bound=worst[0], where=worst[1])
    stats["worst"] = max(stats["worst"], worst[0])
    key = (pr.name, pr.af)
    stats["table"][key] = max(stats["table"].get(key, 0.0), worst[0])
    assert worst[0] <= 1.0, row
    # exact routing: targets in the kernel's order of attended rows
    er = route_exponent(dh)
    idx = {0, nc - 1}
    p0 = parts[0]
    idx |= {min(g.trows, p0["i1"]) - 1, p0["i1"] - 1, parts[-1]["i0"]}
    if nc > g.trows:
        idx.add(g.trows)
    if ns > 1:
        idx.add(parts[1]["i0"])
    idx = sorted(i for i in idx if 0 <= i < nc)
    targets = [("row", int(pos[i]), i) for i in idx] + ([("current", p, nc)] if cur else [])
    routed = weak = 0
    for label, jpos, i in targets:
        xv = x.copy()
        for b in range(B):
            src = (pr.enc[b, jpos] if pr.af == 6 else pr.x_row(jpos, b)) if label == "row" else x[b]
            xv[b, pr.Aq] = src[pr.Ak]
        got, q, kc, vc = pr.run(p, B, xv, er)
        for b, hs in enumerate(oracle_heads(pr, B, pos, cur, q, kc, vc, parts, with_bound=False)):
            for h, (_, _, K, V) in enumerate(hs):
                s, _, _ = da.attend64(q[b, h * dh:(h + 1) * dh], K, V, g.scale2)
                others = np.delete(s, i)
                assert np.isfinite(s).all(), (row, label, jpos, b, h)
                tail = np.exp(others - s[i]).sum() * np.abs(V).max() if len(others) else 0.0
                if len(others) and (s[i] - others.max() < 40 or tail >= 2.0 ** -26):
                    weak += 1            # a key of small norm: the margin the exact check relies on does not hold
                    continue
                want = V[i]
                assert np.array_equal(got[b, h * dh:(h + 1) * dh], want.astype(np.float32)), \
                    dict(row, target=label, position=jpos, index=i, b=b, h=h)
                routed += 1
    row.update(routed_exact=routed, routing_margin_too_small=weak)
    assert weak <= max(1, routed // 20), row
    # negative routing: rows the pattern must not attend, another sample, another head
    negs = []
    pm = p % g.bc
    if pr.af == 1 and p >= g.bc:
        negs.append(("previous block", p - pm - 1, 0, 0))
    if pr.af == 3:
        negs.append(("current block", p, 0, 0))
        if pm > 0:
            negs.append(("current block", p - 1, 0, 0))
    if pr.af == 7 and p >= g.prime_pad:
        negs.append(("current token past the prime", p, 0, 0))
        if p - 1 >= g.prime_pad:
            negs.append(("row past the prime", p - 1, 0, 0))
    if B > 1:
        negs.append(("another sample", int(pos[0]), 1, 0))
    if g.H > 1:
        negs.append(("another head", int(pos[0]), 0, 1))
    aliased = {}
    for label, jpos, db, dhd in negs:
        xv = x.copy()
        srcv = {}
        for b in range(B):
            bs = (b + db) % B
            src = x[bs] if jpos == p else (pr.enc[bs, jpos] if pr.af == 6 else pr.x_row(jpos, bs))
            xv[b, pr.Aq] = src[np.roll(pr.Ak.reshape(g.H, dh), -dhd, axis=0).reshape(-1)]
            if jpos != p:
                srcv[b] = pr.VE[bs, jpos] if pr.af == 6 else pr.V[bs, jpos]
        got, q, kc, vc = pr.run(p, B, xv, er)
        if jpos == p:            # the current token's own v, as this step computed it
            srcv = {b: vc[(b + db) % B] for b in range(B)}
        n_alias = 0
        for b, hs in enumerate(oracle_heads(pr, B, pos, cur, q, kc, vc, parts)):
            for h, (bd, a, _, _) in enumerate(hs):
                o = got[b, h * dh:(h + 1) * dh]
                assert (np.abs(o - a) <= bd).all(), dict(row, negative=label, b=b, h=h)
                hv = (h + dhd) % g.H
                wrong = srcv[b][hv * dh:(hv + 1) * dh].astype(np.float32)
                if (np.abs(wrong - a) <= bd).all():
                    # rows are rotations of shared base rows: another head's key (a rotation by dh) can be an attended
                    # key of this head too, and then the right answer is that value
                    n_alias += 1
                    continue
                assert not np.array_equal(o, wrong), dict(row, negative=label, b=b, h=h)
        assert n_alias <= B * g.H // 4, dict(row, negative=label, aliased=n_alias)
        aliased[label] = aliased.get(label, 0) + n_alias
    row["negatives"] = [n[0] for n in negs]
    row["negatives_aliased"] = aliased
    row["seconds"] = round(time.time() - t_start, 2)
    # leave the caches as the fill made them
    pr.eng.reset(p)
    pr.eng.step(B, x_in=pr.X[p])
    record(row)


def run_case(af, name, depth=1, t_end=None, batch_list=None, windows=1):
    t0 = time.time()
    pr = Probe(af, name, depth)
    g = pr.g
    t_end = t_end or g.n_ctx
    stats = dict(worst=0.0, table={})
    for B in batch_list or batches(g, af, pr.maxb):
        for w in range(windows):
            last = w == windows - 1
            pr.loaded = None
            pr.load(0)                           # before make_rows: set_encoder_kv multiplies by the loaded c_enc_kv
            pr.make_rows(B, seed=100 * B + 7 * af + w)
            pr.eng.reset(0)
            cache = da.CacheRows(g, af)
            probes = set(probe_positions(g, af, B, t_end)) if last else set()
            for p in range(t_end if last else min(t_end, 3 * g.bc + 5)):
                if p in probes:
                    kind, pos, cur = cache.read(p)
                    want_kind, want = da.expected_rows(g, af, p)
                    assert kind == want_kind and (kind == "zeros" or np.array_equal(np.sort(pos), want))
                    assert kind == "zeros" or (pos >= 0).all()
                    check_probe(pr, B, p, pos, cur, kind, stats)
                else:
                    pr.eng.step(B, x_in=pr.X[p])
                cache.write(p)
            torch.cuda.synchronize()
    record(dict(case="summary", geometry=name, pattern=af, depth=depth, windows=windows, RC=g.RC, G=g.G,
                batches=batch_list or batches(g, af, pr.maxb), max_err_over_bound=stats["worst"],
                seconds=round(time.time() - t0, 1)))
    del pr
    torch.cuda.empty_cache()


@pytest.mark.parametrize("af, name", CASES)
def test_attention_probe(af, name):
    run_case(af, name)


def test_depth2_layer1_probe():
    """layer 0 zero, layer 1 the probe: layer 1's cache addressing and flags"""
    run_case(1, "1b", depth=2, t_end=3 * 134 + 3, batch_list=[16])


@pytest.mark.parametrize("af", [1, 3])
def test_second_window_reads_no_stale_rows(af):
    """a window, reset(0), then a window of new rows: the ring rows of the first must never be read"""
    run_case(af, "1b", t_end=3 * 134 + 3, batch_list=[16], windows=2)


def geom_of(af, name, G):
    """the restated geometry of a case's engine, with the plan's tile rows"""
    W, H, n_ctx, blocks, prime, enc, maxb = GEOM[name]
    cfg = prior_config(width=W, depth=1, heads=H, n_state=W // 4, mlp_width=W, n_ctx=n_ctx, blocks=blocks,
                       attn_funcs=[af], bins=0, prime_len=prime, encoder_dims=enc, max_batch=maxb)
    return da.Geom(heads=H, dh=W // 4 // H, n_ctx=n_ctx, blocks=blocks, prime_len=prime, enc_dims=enc, G=G,
                   RC=tile_rows(cfg, G))


def case_features(g, af, B):
    """what the probes of one case visit, from the restated partition (the same positions run_case checks)"""
    out = defaultdict(set)
    for p in probe_positions(g, af, B, g.n_ctx):
        R, _, cur, _ = da.attn_geom(g, af, p)
        if R == 0:
            continue
        nc = da.ncache_of(R, cur)
        ns = da.attn_nsplit(g, da.gmax_of(g, B), nc)
        parts = da.partition(g, nc, ns, cur)
        _, nr, wc = parts[-1]["tiles"][-1]
        out["ns"].add(ns)
        out["tiles per part >= 3"].add(max(len(pt["tiles"]) for pt in parts) >= 3)
        out["full last tile"].add(nr + wc == g.RC)
        out["items not prefetched"].add(any(not i["prefetched"] for i in da.items(g, B, ns, R)))
        out["rows kernel"].add(16 if B <= 16 else 32)
        out["K/V tile"].add("swizzled" if g.swizzled else "linear")
    return out


def test_coverage():
    """what the cases above visit (their probe positions, restated): every split, parts of 3 tiles or more, a full last
    tile, items that were not prefetched, both row kernels, swizzled and linear tiles"""
    G = sm_count()
    cover = defaultdict(set)
    for af, name in CASES:
        g = geom_of(af, name, G)
        for B in batches(g, af, GEOM[name][-1]):
            for k, v in case_features(g, af, B).items():
                cover[k] |= v
    record(dict(case="coverage", G=G, device=torch.cuda.get_device_name(),
                **{k: sorted(v, key=str) for k, v in cover.items()}))
    assert cover["ns"] >= {1, 2, 3, 4}
    assert True in cover["tiles per part >= 3"]
    assert True in cover["full last tile"]
    assert True in cover["items not prefetched"]
    assert cover["rows kernel"] == {16, 32}
    assert cover["K/V tile"] == {"swizzled", "linear"}
