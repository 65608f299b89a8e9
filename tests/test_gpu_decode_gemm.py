"""The decode step's four Conv1D phases (csrc/decode_engine.cu gemm_phase<R>) against float64 at the priors' real
geometry, through every K split, column plan, warp dealing and row tile the device's plans contain.

Probe layers on a DecodeEngine (bins = 0, x_in fed, h_out read).  Only the probed layer is nonzero; a zero layer passes
x through exactly.  The probed layer's pattern is 2 (transpose) with n_ctx 16 and 4 blocks: positions 0 .. 3 attend only
themselves (softmax exactly 1, the attention output is the kernel's own v), later positions attend 2 .. 4 cached rows.

a. Exact probes, bit for bit.  LayerNorm gamma is small and beta about +-1 (oracle.decode_gemm.exact_ln), so the staged
   rows (oracle.decode_stats.staged, row dependent) are fp16 values on a coarse enough grid; the probed Conv1D has
   sparse weights on {-7..7} 2^-3 (every k-step of every unit meets one) and a grid bias; the other Conv1Ds select or
   are zero.  Every partial sum in any order is then an fp32 value (asserted: decode_gemm.exact_in_fp32), so the
   kernel must return fp16(s64 + b) through its epilogue bit for bit:
     qkv  the V third, observed through single-key attention and a selection c_proj: h[:, Bc] = fp16(x + v)
     proj a selection of LN0 as v, proj the probe:                               h = fp16(x + y)
     fc   fc the probe, quick_gelu16, a selection proj2:                         h[:, perm] = fp16(x + g)
          (quick_gelu may be one fp16 ulp off where the oracle flags its float32 value near a rounding boundary)
     proj2 a selection fc of LN1 values in {0} u [8, 16), where quick_gelu16 is the identity (asserted), proj2 the probe
   and h = x on every column the probe does not reach.
b. Rounding probes: real LayerNorm inputs (oracle.synth gamma / beta, N(0, 1) rows) and dense weights of oracle.synth's
   scale times 2^e: every observed element must lie in decode_gemm.admissible's range (the fp16 values that round
   from the float64 result +- its bound, carried through the same epilogues); fp32 weights everywhere, and fp16
   weights and biases at the 5b width.  proj2's input is quick_gelu16 of real LN1 values (fc a selection); where the
   oracle flags that the device may round one of them the other way, the bound is widened by the effect of that ulp
   (check_step).  The fraction that needed the neighbour is recorded.
c. The Q and K thirds through attention at positions 4 .. 15 (2, 3 or 4 keys): exact-probe Q and K weights (q and k
   are then exactly the float64 GEMM's, fp16(s64 + b), so the admissible set is one value and
   oracle.decode_attn.bound needs no extension for them), v a selection of LN0, x = 0 on Bc; h[:, Bc] must be within
   the attention bound.  At an attn_func 6 layer (5b_lyrics' encoder-decoder layers, whose QKV is Q alone: the only
   layers with 1 and 2 QKV column groups per unit at that width) the exact-probe Q attends the 512 encoder rows, K and
   V fp16 random rows set through a selection c_enc_kv, against the same bound.

Every case runs consecutive steps (positions 0 ..), then a second window after reset(0), so the exchange flags of
several launches are exercised.  Depth and probed layers come from the device's plan (plan_probes): the probed layers
cover every (Conv1D, ncg, in_order, two_rows, nkk < 8, KS) combination of the full-size plan (test_coverage).  Batches
1, 16, 17, 32 and the engine's max batch, up to that max batch (5b: 1 and 16; its 8-row layout: 1 and 8).  One JSON line per case
(pytest -s)."""
import ctypes as C
import json
import time
import zlib
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from jukebox_b200 import _lib
from jukebox_b200.engine import DecodeEngine, prior_config
from jukebox_b200.transformer.transformer import attn_func_of
from oracle import decode_attn as da
from oracle import decode_gemm as dg
from oracle.decode_stats import quick_gelu16, staged
from oracle.synth import synth_tensor

pytestmark = pytest.mark.gpu

# name: (full-size configuration of tests/test_decode_plan_cpu.py or None, width, heads, n_state, max batch of the probe
# engine).  1104 / 272: a width that is not a multiple of 64 (K split 1, units with one or no QKV column group)
GEOM = {"1b": ("1b_lyrics", 2048, 2, 512, 32), "5b": ("5b_lyrics", 4800, 8, 1200, 16),
        "up": ("upsampler_level_0", 1920, 1, 480, 32), "small_up": ("small_upsampler", 1024, 1, 256, 32),
        "1104": (None, 1104, 1, 272, 32),
        # the 8-row layout leaves 5b_lyrics a deeper weight ring: its proj phase fits it there (not in_order)
        "5b_8": ("5b_lyrics", 4800, 8, 1200, 8)}
FULL = {   # width, depth, heads, attn_order, max_batch of the full-size plans (tests/test_decode_plan_cpu.py CONFIGS)
    "1b_lyrics": (2048, 72, 2, 12, 16), "5b_lyrics": (4800, 79, 8, 10, 8), "small_upsampler": (1024, 48, 1, 2, 16),
    "upsampler_level_0": (1920, 72, 1, 2, 16)}
BATCHES = (1, 16, 17, 32)
N_CTX, BLOCKS = 16, 4
ENC = 512
KINDS = ("qkv", "proj", "fc", "proj2")


def record(row):
    print(json.dumps(row))


def sm_count():
    out = C.c_int(0)
    _lib.check(_lib.lib().jk_device_sm_count(C.byref(out)))
    return out.value


# ---- plans ---------------------------------------------------------------------------------------------------------
def plan_of(cfg, G):
    info = _lib.PlanInfo()
    _lib.check(_lib.lib().jk_prior_plan(C.byref(cfg), G, C.byref(info), None, 0))
    cols = (C.c_uint16 * (2 * G * cfg.depth * 4 * 2 + 64))()
    _lib.check(_lib.lib().jk_prior_plan(C.byref(cfg), G, C.byref(info), cols, len(cols)))
    U = info.units
    arr = np.frombuffer(cols, np.uint16)[:U * cfg.depth * 8].reshape(U, cfg.depth, 4, 2).astype(np.int64)
    return info, arr


def k_of(cfg):
    return [cfg.width, cfg.n_state, cfg.width, cfg.mlp_width]


def combos(cfg, info, cols, layers, gis=range(4)):
    """{(Conv1D, ncg, in_order, two_rows, nkk < 8, KS)} of the given layers (ncg 0: a count-only unit)"""
    out = set()
    for l in layers:
        for gi in gis:
            for ncg in set(int(n) for n in cols[:, l, gi, 1]):
                if ncg == 0:
                    out.add((KINDS[gi], 0, None, None, None, info.k_split))
                    continue
                ph = dg.Phase(k_of(cfg)[gi], info.k_split, ncg, info.ring_slots)
                out.add((KINDS[gi], ncg, ph.in_order, ph.two_rows, ph.nkk < 8, info.k_split))
    return out


def full_config(name):
    W, depth, H, order, mb = FULL[name]
    afs = [attn_func_of(order, d) for d in range(depth)]
    return prior_config(width=W, depth=depth, heads=H, n_state=W // 4, mlp_width=W, n_ctx=8192, blocks=128,
                        attn_funcs=afs, bins=0, encoder_dims=ENC if 6 in afs else 0, max_batch=mb), afs


def probe_config(geo, depth, afs_full):
    full, W, H, S, mb = GEOM[geo]
    afs = [6 if a == 6 else 2 for a in afs_full[:depth]]
    return prior_config(width=W, depth=depth, heads=H, n_state=S, mlp_width=W, n_ctx=N_CTX, blocks=BLOCKS,
                        attn_funcs=afs, bins=0, encoder_dims=ENC if 6 in afs else 0, max_batch=mb), afs


def plan_probes(geo, G):
    """(probe config, attn funcs, probed layers, target combinations, uncovered) for one geometry on G SMs: the target
    is every combination of the full-size plan (the Q-only QKV of its attn_func 6 layers included), the depth the
    shortest prefix of the full stack whose layers reach all of them, the probed layers a greedy cover"""
    full = GEOM[geo][0]
    if full is None:
        cfg, afs = probe_config(geo, 2, [2, 2])
        info, cols = plan_of(cfg, G)
        return cfg, afs, [0, 1], combos(cfg, info, cols, [0, 1]), set()
    fcfg, fafs = full_config(full)
    finfo, fcols = plan_of(fcfg, G)
    target = set()
    for l in range(fcfg.depth):
        target |= combos(fcfg, finfo, fcols, [l])
    pairs = lambda cs: {c[:2] for c in cs}      # in_order depends on the ring, i.e. on the engine's max batch
    for depth in range(1, fcfg.depth + 1):
        cfg, afs = probe_config(geo, depth, fafs)
        info, cols = plan_of(cfg, G)
        per = {l: combos(cfg, info, cols, [l]) for l in range(depth)}
        have = set().union(*per.values()) if per else set()
        if pairs(target) <= pairs(have) or depth == fcfg.depth:
            break
    chosen, got = [], set()
    while True:
        l = max(per, key=lambda k: len((per[k] & target) - got) + len(pairs(per[k]) - pairs(got)))
        if not (per[l] & target) - got and not pairs(per[l]) - pairs(got):
            break
        chosen.append(l)
        got |= per[l]
    if 0 not in chosen:
        chosen.append(0)
    return cfg, afs, sorted(chosen), target, target - got


GI = {"qkv": 0, "qk": 0, "q6": 0, "proj": 1, "fc": 2, "proj2": 3}


def schedule(afs, layers):
    """the probes test_conv1d_probes runs, as (layer, probe, mode).  proj and proj2 columns are one assignment for the
    whole stack: their probes, and the rounding probes, run in the first probed layer (never attn_func 6: the exact
    probes carry the other layers' column plans).  A layer of attn_func 6 has a Q-only QKV: its Q goes through
    attention over the encoder rows ("q6"); elsewhere the V third is probed directly and Q and K through attention
    over cached rows ("qk")."""
    first = layers[0]
    assert afs[first] != 6
    out = []
    for l in layers:
        if afs[l] == 6:
            out += [(l, "fc", "exact"), (l, "q6", "exact")]
            continue
        out += [(l, k, "exact") for k in (KINDS if l == first else ("qkv", "fc"))]
        if l == first:
            out += [(l, k, "round") for k in KINDS]
        out.append((l, "qk", "exact"))
    return out


# ---- probe layers --------------------------------------------------------------------------------------------------
class Probe:
    """one geometry's engine (zero layers everywhere but the probe) and the numpy model of its probes"""

    def __init__(self, geo, G, seed=0):
        self.geo = geo
        self.cfg, self.afs, self.layers, self.target, self.uncovered = plan_probes(geo, G)
        c = self.cfg
        self.W, self.S, self.H, self.depth = c.width, c.n_state, c.heads, c.depth
        self.mb = GEOM[geo][4]
        self.info, self.cols = plan_of(c, G)
        self.eng = DecodeEngine(width=c.width, depth=c.depth, heads=c.heads, n_state=c.n_state, mlp_width=c.mlp_width,
                                n_ctx=N_CTX, blocks=BLOCKS, attn_funcs=list(self.afs), bins=0,
                                encoder_dims=c.encoder_dims, max_batch=self.mb)
        for l in range(self.depth):
            self.eng.load_layer(l, self.zero_block(self.afs[l]))
        rng = np.random.default_rng(500 + seed)
        perm = rng.permutation(self.W)
        S = self.S
        self.Aq, self.Ak, self.Av, self.Bc = perm[:S], perm[S:2 * S], perm[2 * S:3 * S], perm[3 * S:4 * S]
        self.perm = rng.permutation(self.W)          # fc column j -> residual column perm[j] (probe fc)
        self.sel = rng.permutation(self.W)           # fc column j = LN1 column sel[j] (probe proj2)
        self.G = G
        self.zero_encoder()
        self.g = da.Geom(heads=self.H, dh=S // self.H, n_ctx=N_CTX, blocks=BLOCKS, enc_dims=c.encoder_dims, G=G,
                         RC=self.info.tile_rows)

    def zero_encoder(self):
        """encoder K / V of every attn_func 6 layer from zero rows: zero, so a zero layer's attention outputs 0"""
        if self.cfg.encoder_dims:
            self.eng.set_encoder_kv(torch.zeros(self.mb, self.cfg.encoder_dims, self.W, device="cuda"))

    def zero_block(self, af=2, dtype=torch.float32):
        W, S = self.W, self.S
        z = lambda *s: torch.zeros(*s, device="cuda", dtype=dtype)
        blk = NS(attn=NS(attn_func=af, c_attn=NS(w=z(W, S if af == 6 else 3 * S), b=z(S if af == 6 else 3 * S)),
                         c_proj=NS(w=z(S, W), b=z(W))),
                 mlp=NS(c_fc=NS(w=z(W, W), b=z(W)), c_proj=NS(w=z(W, W), b=z(W))),
                 ln_0=NS(weight=torch.ones(W, device="cuda"), bias=torch.zeros(W, device="cuda")),
                 ln_1=NS(weight=torch.ones(W, device="cuda"), bias=torch.zeros(W, device="cuda")))
        if af == 6:
            blk.attn.c_enc_kv = NS(w=z(W, 2 * S), b=z(2 * S))
        return blk

    def phases(self, l, gi):
        """{ncg: columns} of Conv1D gi in layer l, and {ncg: Phase}"""
        groups = dg.unit_groups(self.cols[:, l, gi])
        return groups, {n: dg.Phase(k_of(self.cfg)[gi], self.info.k_split, n, self.info.ring_slots) for n in groups}


def build(pr, kind, mode, rng, e=0, dtype=torch.float32, af=2):
    """(numpy model, torch block) of one probe: kind in KINDS, "qk" or "q6"; mode "exact" or "round"; af the layer's
    attn_func (6: a Q-only c_attn and c_enc_kv)"""
    W, S = pr.W, pr.S
    j = np.arange(S)
    m = NS(kind=kind, mode=mode)
    if mode == "exact":
        m.g0, m.b0 = dg.exact_ln(rng, W)
    else:
        m.g0 = synth_tensor("_attn_mods.0.ln_0.weight", (W,), 3)
        m.b0 = synth_tensor("_attn_mods.0.ln_0.bias", (W,), 3)
    if kind == "proj2" and mode == "exact":
        m.g1, m.b1 = dg.identity_gelu_ln(rng, W)
    elif kind == "proj2":
        m.g1 = synth_tensor("_attn_mods.0.ln_1.weight", (W,), 3)
        m.b1 = synth_tensor("_attn_mods.0.ln_1.bias", (W,), 3)
    else:
        m.g1, m.b1 = m.g0, m.b0
    aw, ab = np.zeros((W, S if af == 6 else 3 * S), np.float32), np.zeros(S if af == 6 else 3 * S, np.float32)
    ew = np.zeros((W, 2 * S), np.float32)
    pw, pb = np.zeros((S, W), np.float32), np.zeros(W, np.float32)
    fw, fb = np.zeros((W, W), np.float32), np.zeros(W, np.float32)
    qw, qb = np.zeros((W, W), np.float32), np.zeros(W, np.float32)

    def probe_w(K, N, name):
        if mode == "exact":
            return dg.grid_weights(rng, K, N), dg.grid_bias(rng, N)
        return (synth_tensor(f"_attn_mods.0.{name}.w", (K, N), 5) * np.float32(2.0 ** e),
                synth_tensor(f"_attn_mods.0.{name}.b", (N,), 5) * np.float32(2.0 ** e))

    if kind == "qkv":
        aw[:, 2 * S:], ab[2 * S:] = probe_w(W, S, "attn.c_attn")
        pw[j, pr.Bc] = 1.0
    elif kind == "proj":
        aw[pr.Av, 2 * S + j] = 1.0
        pw[:], pb[:] = probe_w(S, W, "attn.c_proj")
    elif kind == "fc":
        fw[:], fb[:] = probe_w(W, W, "mlp.c_fc")
        qw[np.arange(W), pr.perm] = 1.0
    elif kind == "proj2":
        fw[pr.sel, np.arange(W)] = 1.0
        qw[:], qb[:] = probe_w(W, W, "mlp.c_proj")
    elif kind == "qk":
        aw[:, :S], ab[:S] = dg.grid_weights(rng, W, S), dg.grid_bias(rng, S)
        aw[:, S:2 * S], ab[S:2 * S] = dg.grid_weights(rng, W, S), dg.grid_bias(rng, S)
        aw[pr.Av, 2 * S + j] = 1.0
        pw[j, pr.Bc] = 1.0
    elif kind == "q6":
        assert af == 6
        aw[:], ab[:] = dg.grid_weights(rng, W, S), dg.grid_bias(rng, S)
        ew[pr.Ak, j] = 1.0                      # encoder K = fp16(enc[:, :, Ak]), V = fp16(enc[:, :, Av])
        ew[pr.Av, S + j] = 1.0
        pw[j, pr.Bc] = 1.0
    m.aw, m.ab, m.pw, m.pb, m.fw, m.fb, m.qw, m.qb = aw, ab, pw, pb, fw, fb, qw, qb
    t = lambda a: torch.from_numpy(a).to("cuda", dtype)
    blk = NS(attn=NS(attn_func=af, c_attn=NS(w=t(aw), b=t(ab)), c_proj=NS(w=t(pw), b=t(pb))),
             mlp=NS(c_fc=NS(w=t(fw), b=t(fb)), c_proj=NS(w=t(qw), b=t(qb))),
             ln_0=NS(weight=torch.from_numpy(m.g0).cuda(), bias=torch.from_numpy(m.b0).cuda()),
             ln_1=NS(weight=torch.from_numpy(m.g1).cuda(), bias=torch.from_numpy(m.b1).cuda()))
    if af == 6:
        blk.attn.c_enc_kv = NS(w=t(ew), b=t(np.zeros(2 * S, np.float32)))
    return m, blk


def probe_operands(pr, m, x):
    """(A, W, b, gi, observed h columns, input uncertainty) of the probed Conv1D for fp16 rows x.  The input
    uncertainty (proj2's rounding probe only, else None) is per input element the distance to the farther fp16
    neighbour where quick_gelu16 flags that the device may round fc's output the other way, 0 elsewhere."""
    W, S = pr.W, pr.S
    if m.kind in ("qkv", "proj", "qk"):
        A0 = staged(x, m.g0, m.b0)
        if m.kind == "qkv":                   # the whole Conv1D (its plan), the V third observed
            return A0, m.aw, m.ab, 0, pr.Bc, None
        return A0[:, pr.Av], m.pw, m.pb, 1, np.arange(W), None
    A1 = staged(x, m.g1, m.b1)
    if m.kind == "fc":
        return A1, m.fw, m.fb, 2, pr.perm, None
    g, near = quick_gelu16(A1[:, pr.sel])       # fc is a selection: its output is LN1, proj2's input quick_gelu of it
    if m.mode == "exact":
        assert np.array_equal(g, A1[:, pr.sel]) and not near.any(), "proj2 probe: quick_gelu16 is not the identity"
        return g, m.qw, m.qb, 3, np.arange(W), None
    gap = np.maximum(np.abs(np.nextafter(g, np.float16(np.inf)).astype(np.float64) - g),
                     np.abs(g - np.nextafter(g, np.float16(-np.inf)).astype(np.float64)))
    return g, m.qw, m.qb, 3, np.arange(W), np.where(near, gap, 0.0)


def check_step(pr, m, l, x, got, stats):
    """got: h_out [B, W] of one step, x its fp16 rows: the probed Conv1D's outputs in the admissible set, x elsewhere"""
    A, Wt, b, gi, obs, gap = probe_operands(pr, m, x)
    W16, b32 = dg.weights16(Wt), dg.bias32(b)
    groups, phases = pr.phases(l, gi)
    if m.mode == "exact":
        assert dg.exact_in_fp32(A, W16, b32), "probe operands are not exact in fp32"
        sb = dg.conv64(A, W16, b32)
        bd = np.zeros(sb.shape)
    else:
        sb, bd = dg.conv_bound(A, W16, b32, groups, phases)
        if gap is not None:
            # the kernel multiplies its own quick_gelu outputs, each within `gap` of A: that moves s by at most
            # gap . |W|, and the rounding terms evaluated at those inputs by 17 u n (gap . |W|) << gap . |W| (n the
            # k-steps of a warp), so twice gap . |W| covers both
            bd = bd + 2 * (gap @ np.abs(W16.astype(np.float64)))
    if gi == 0:
        sb, bd = sb[:, 2 * pr.S:], bd[:, 2 * pr.S:]
    lo, hi, near, n = dg.admissible("fc" if gi == 2 else "qkv", sb, bd, x=x[:, obs])
    ok = dg.in_interval(got[:, obs], lo, hi)
    rest = np.setdiff1d(np.arange(pr.W), obs)
    stray = int((got[:, rest] != x[:, rest].astype(np.float32)).sum())
    nearest = got[:, obs] == near.astype(np.float32)
    stats["elements"] += ok.size
    stats["mismatches"] += int((~ok).sum())
    stats["stray"] += stray
    stats["needed_neighbour"] += int((ok & ~nearest).sum())
    stats["candidates_max"] = max(stats["candidates_max"], int(n.max()))
    stats["several_candidates"] += int((n > 1).sum())
    if (~ok).any() and len(stats["bad"]) < 5:
        i, c = np.argwhere(~ok)[0]
        stats["bad"].append(dict(layer=l, row=int(i), col=int(obs[c]), got=float(got[i, obs[c]]),
                                 want=float(near[i, c]), lo=float(lo[i, c]), hi=float(hi[i, c]),
                                 B=x.shape[0]))


def run_probe(pr, l, kind, mode, batches, e=0, dtype=torch.float32, seed=0):
    rng = np.random.default_rng(seed)
    m, blk = build(pr, kind, mode, rng, e, dtype, af=pr.afs[l])
    pr.eng.load_layer(l, blk)
    stats = dict(elements=0, mismatches=0, stray=0, needed_neighbour=0, several_candidates=0, candidates_max=0, steps=0,
                 bad=[])
    for B in batches:
        for window, steps in (((0, 3), (1, 1)) if mode == "exact" else ((0, 2), (1, 1))):
            pr.eng.reset(0)
            for p in range(steps):
                if mode == "exact":
                    x = dg.grid_rows(rng, B, pr.W).astype(np.float16)
                else:
                    x = rng.standard_normal((B, pr.W)).astype(np.float16)
                h = torch.full((B, pr.W), float("nan"), device="cuda")
                pr.eng.step(B, x_in=torch.from_numpy(x.astype(np.float32)).cuda(), h_out=h)
                check_step(pr, m, l, x, h.cpu().numpy(), stats)
                stats["steps"] += 1
    pr.eng.load_layer(l, pr.zero_block(pr.afs[l]))
    return stats


def run_qk(pr, l, batches, seed=0):
    """part c: q and k of the exact probe through attention at positions 4 .. 15 (2, 3 and 4 keys)"""
    rng = np.random.default_rng(seed)
    m, blk = build(pr, "qk", "exact", rng)
    pr.eng.load_layer(l, blk)
    W, S, g, dh = pr.W, pr.S, pr.g, pr.g.dh
    worst, checked, nonexact = 0.0, 0, 0
    for B in batches:
        pr.eng.reset(0)
        cache = da.CacheRows(g, 2)
        Ks, Vs = {}, {}
        for p in range(N_CTX):
            x = dg.grid_rows(rng, B, W)
            x[:, pr.Bc] = 0
            x = x.astype(np.float16)
            A0 = staged(x, m.g0, m.b0)
            q = []
            for cols, bias in ((slice(0, S), m.ab[:S]), (slice(S, 2 * S), m.ab[S:2 * S])):
                w16, b32 = dg.weights16(m.aw[:, cols]), dg.bias32(bias)
                if not dg.exact_in_fp32(A0, w16, b32):
                    nonexact += 1
                q.append(dg.f16(dg.conv64(A0, w16, b32)))
            q, k, v = q[0], q[1], A0[:, pr.Av]
            Ks[p], Vs[p] = k, v
            h = torch.full((B, W), float("nan"), device="cuda")
            pr.eng.step(B, x_in=torch.from_numpy(x.astype(np.float32)).cuda(), h_out=h)
            got = h.cpu().numpy()
            rest = np.setdiff1d(np.arange(W), pr.Bc)
            assert (got[:, rest] == x[:, rest].astype(np.float32)).all(), (pr.geo, l, p, "columns outside Bc")
            kind, pos, cur = cache.read(p)
            ns = da.attn_nsplit(g, da.gmax_of(g, B), len(pos) - cur)
            parts = da.partition(g, len(pos) - cur, ns, cur)
            for b in range(B):
                K = np.stack([Ks[t][b] for t in pos])
                V = np.stack([Vs[t][b] for t in pos])
                for hh in range(g.H):
                    sl = slice(hh * dh, (hh + 1) * dh)
                    bd, a, _ = da.bound(q[b, sl], K[:, sl], V[:, sl], g, parts)
                    r = np.abs(got[b, pr.Bc[sl]] - a) / bd
                    worst = max(worst, float(r.max()))
                    checked += 1
                    assert (r <= 1).all(), dict(geometry=pr.geo, layer=l, p=p, B=B, b=b, h=hh, err_over_bound=float(r.max()))
            cache.write(p)
    assert nonexact == 0, "qk probe operands are not exact in fp32"
    pr.eng.load_layer(l, pr.zero_block(pr.afs[l]))
    return dict(max_err_over_bound=worst, heads_checked=checked)


def run_q6(pr, l, batches, seed=0):
    """part c at an attn_func 6 layer: the Q-only QKV of the exact probe through attention over the encoder rows
    (K, V = fp16 of random encoder rows through a selection c_enc_kv), positions 0 .. 3"""
    rng = np.random.default_rng(seed)
    m, blk = build(pr, "q6", "exact", rng, af=6)
    pr.eng.load_layer(l, blk)
    W, S, g, dh = pr.W, pr.S, pr.g, pr.g.dh
    E = pr.cfg.encoder_dims
    worst, checked = 0.0, 0
    w16, b32 = dg.weights16(m.aw), dg.bias32(m.ab)
    for B in batches:
        enc = rng.standard_normal((B, E, W)).astype(np.float16)
        pr.eng.set_encoder_kv(torch.from_numpy(enc.astype(np.float32)).cuda())
        KE, VE = enc[:, :, pr.Ak], enc[:, :, pr.Av]
        ns = da.attn_nsplit(g, da.gmax_of(g, B), E)
        parts = da.partition(g, E, ns, 0)
        pr.eng.reset(0)
        for p in range(4):
            x = dg.grid_rows(rng, B, W)
            x[:, pr.Bc] = 0
            x = x.astype(np.float16)
            A0 = staged(x, m.g0, m.b0)
            assert dg.exact_in_fp32(A0, w16, b32), "q6 probe operands are not exact in fp32"
            q = dg.f16(dg.conv64(A0, w16, b32))
            h = torch.full((B, W), float("nan"), device="cuda")
            pr.eng.step(B, x_in=torch.from_numpy(x.astype(np.float32)).cuda(), h_out=h)
            got = h.cpu().numpy()
            rest = np.setdiff1d(np.arange(W), pr.Bc)
            assert (got[:, rest] == x[:, rest].astype(np.float32)).all(), (pr.geo, l, p, "columns outside Bc")
            for b in range(B):
                for hh in range(g.H):
                    sl = slice(hh * dh, (hh + 1) * dh)
                    bd, a, _ = da.bound(q[b, sl], KE[b][:, sl], VE[b][:, sl], g, parts)
                    r = np.abs(got[b, pr.Bc[sl]] - a) / bd
                    worst = max(worst, float(r.max()))
                    checked += 1
                    assert (r <= 1).all(), dict(geometry=pr.geo, layer=l, p=p, B=B, b=b, h=hh, err_over_bound=float(r.max()))
    pr.eng.load_layer(l, pr.zero_block(6))
    pr.zero_encoder()
    return dict(max_err_over_bound=worst, heads_checked=checked, encoder_rows=E)


def batches_of(mb):
    """BATCHES up to the engine's max batch, and the max batch itself (5b_8: 1 and 8)"""
    return sorted({B for B in BATCHES if B <= mb} | {mb})


def seed_of(*key):
    return zlib.crc32(repr(key).encode()) % 100000


CASES = list(GEOM)


@pytest.mark.parametrize("geo", CASES)
def test_conv1d_probes(geo):
    t0 = time.time()
    G = sm_count()
    pr = Probe(geo, G)
    batches = batches_of(pr.mb)
    summary = dict(case="summary", geometry=geo, G=G, depth=pr.depth, K_split=pr.info.k_split,
                   ring_slots=pr.info.ring_slots, probed_layers=pr.layers, batches=batches,
                   skipped_batches=[B for B in BATCHES if B > pr.mb], neighbour=0, elements=0, qk_worst=0.0)
    for l, kind, mode in schedule(pr.afs, pr.layers):
        ts = time.time()
        if kind in ("qk", "q6"):
            res = (run_qk if kind == "qk" else run_q6)(pr, l, batches, seed=seed_of(geo, l, kind))
            record(dict(geometry=geo, layer=l, attn_func=pr.afs[l],
                        conv1d="qkv: Q and K through attention" if kind == "qk" else "Q-only qkv through encoder attention",
                        ncg=sorted(set(int(n) for n in pr.cols[:, l, 0, 1])), **res, seconds=round(time.time() - ts, 2)))
            summary["qk_worst"] = max(summary["qk_worst"], res["max_err_over_bound"])
            continue
        for dtype in ((torch.float32, torch.float16) if (mode == "round" and geo == "5b") else (torch.float32,)):
            ts = time.time()
            e = 2 if mode == "round" and kind == "proj" else 0
            st = run_probe(pr, l, kind, mode, batches, e=e, dtype=dtype, seed=seed_of(geo, l, kind, mode))
            row = dict(geometry=geo, layer=l, attn_func=pr.afs[l], conv1d=kind, probe=mode,
                       weights=str(dtype).split(".")[-1], ncg=sorted(set(int(n) for n in pr.cols[:, l, GI[kind], 1])),
                       neighbour_fraction=st["needed_neighbour"] / max(1, st["elements"]),
                       seconds=round(time.time() - ts, 2), **{k: v for k, v in st.items() if k != "bad"},
                       first_mismatches=st["bad"])
            record(row)
            assert st["mismatches"] == 0 and st["stray"] == 0, row
            if mode == "round":
                summary["neighbour"] += st["needed_neighbour"]
                summary["elements"] += st["elements"]
    summary["neighbour_fraction"] = summary["neighbour"] / max(1, summary["elements"])
    summary["seconds"] = round(time.time() - t0, 1)
    record(summary)
    del pr
    torch.cuda.empty_cache()


def coverage(G):
    """what test_conv1d_probes visits on G SMs, restated from the plans and the schedule: per geometry the target
    combinations, the visited ones, and per Conv1D the units whose columns a probe observed (every column of a probed
    Conv1D is observed, and each of a unit's K-split CTAs finishes 4 ncg / KS > 0 of its column pairs) against the units
    that own columns of that Conv1D in any layer"""
    out = {}
    for geo in CASES:
        cfg, afs, layers, target, uncovered = plan_probes(geo, G)
        info, cols = plan_of(cfg, G)
        vis, units = set(), {gi: set() for gi in range(4)}
        for l, kind, _ in schedule(afs, layers):
            gi = GI[kind]
            vis |= combos(cfg, info, cols, [l], [gi])
            units[gi] |= {u for u in range(info.units) if cols[u, l, gi, 1] > 0}
        owners = {gi: {u for u in range(info.units) for l in range(cfg.depth) if cols[u, l, gi, 1] > 0}
                  for gi in range(4)}
        out[geo] = dict(target=target, visited=vis, layers=layers, depth=cfg.depth, units=info.units,
                        units_observed={KINDS[gi]: len(units[gi]) for gi in range(4)},
                        units_owning={KINDS[gi]: len(owners[gi]) for gi in range(4)},
                        missing_units={KINDS[gi]: sorted(owners[gi] - units[gi]) for gi in range(4)})
    return out


def test_coverage():
    """every combination of the full-size plans visited (by the engines of that configuration together), the Q-only
    QKV of attn_func 6 layers included; for each Conv1D, every unit (so every CTA) that owns columns of it in some
    layer has its columns observed by a probe"""
    G = sm_count()
    cov = coverage(G)
    by_full = {}
    for geo, c in cov.items():
        record(dict(case="coverage", geometry=geo, G=G, device=torch.cuda.get_device_name(), depth=c["depth"],
                    probed_layers=c["layers"], visited=sorted(map(str, c["visited"])), units=c["units"],
                    units_observed=c["units_observed"], units_owning=c["units_owning"]))
        t, v = by_full.setdefault(GEOM[geo][0] or geo, (set(), set()))
        t |= c["target"]
        v |= c["visited"]
        assert not any(c["missing_units"].values()), (geo, c["missing_units"])
    for name, (t, v) in by_full.items():
        record(dict(case="coverage", full_size=name, combinations=len(t), not_visited=sorted(map(str, t - v))))
        assert t <= v, (name, t - v)
