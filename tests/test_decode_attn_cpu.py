"""oracle/decode_attn.py on the CPU: the restated layout of the decode step's attention against the reference's pattern,
the float64 attention against transformer_np.attend_one, and the error bound against a numpy emulation of the kernel's
arithmetic, including emulations with one deliberate fault each, which the checks must catch."""
import ctypes as C

import numpy as np
import pytest

from jukebox_b200 import _lib
from oracle import decode_attn as da
from oracle.transformer_np import attend_one

# name: (width, heads, n_ctx, blocks, prime_len, encoder rows, patterns).  1b_lyrics, 5b_lyrics, the upsamplers, and a
# width-2048 geometry with 16 heads of 32 dims, so that B * H passes the SM count and CTAs take several items
REAL = {"1b": (2048, 2, 8576, 64, 384, 0, (0, 1, 2, 3, 7)),
        "5b": (4800, 8, 8192, 128, 0, 512, (1, 2, 3, 6)),
        "up": (1920, 1, 8192, 128, 0, 0, (1, 2, 3)),
        "many": (2048, 16, 1024, 16, 0, 0, (0,))}
SMALL = da.Geom(heads=2, dh=24, n_ctx=96, blocks=8, prime_len=12, enc_dims=20, RC=16)


# the tile rows the plan gives these geometries on 132 SMs: attn_tile_rows(dh_pad), halved while the weight ring would
# get fewer than 4 slots (5b_lyrics: K split 1, so its activation tile leaves room for 16-row K / V tiles only)
TILE_ROWS = {"1b": 48, "5b": 16, "up": 16, "many": 64}


def geom(name, G=132):
    W, H, n_ctx, blocks, prime, enc, _ = REAL[name]
    return da.Geom(heads=H, dh=W // 4 // H, n_ctx=n_ctx, blocks=blocks, prime_len=prime, enc_dims=enc, G=G,
                   RC=TILE_ROWS[name])


def layout_mismatches(g, af, mutate=None, positions=None):
    """positions whose attended rows (as the kernel addresses the cache) are not the reference's"""
    cache = da.CacheRows(g, af, mutate)
    bad = []
    for p in range(g.n_ctx):
        kind, pos, cur = cache.read(p)
        want_kind, want = da.expected_rows(g, af, p)
        if positions is None or p in positions:
            if kind != want_kind or (kind == "rows" and not np.array_equal(np.sort(pos), want)):
                bad.append(p)
        cache.write(p)
    return bad


@pytest.mark.parametrize("af", [0, 1, 2, 3, 6, 7])
def test_layout_small_every_position(af):
    assert layout_mismatches(SMALL, af) == []


@pytest.mark.parametrize("name, af", [(n, af) for n in REAL for af in REAL[n][-1]])
def test_layout_real_geometry(name, af):
    assert layout_mismatches(geom(name), af) == []


@pytest.mark.parametrize("mutate, af", [("base+1", 0), ("base+1", 1), ("base+1", 2), ("base+1", 3), ("base+1", 7),
                                        ("transpose_as_p", 2), ("prev_swap", 3)])
def test_layout_mutations_are_caught(mutate, af):
    assert layout_mismatches(SMALL, af, mutate), f"{mutate} on pattern {af} went unnoticed"


def plan_tile_rows(name, max_batch, sms=132):
    W, H, n_ctx, blocks, prime, enc, afs = REAL[name]
    cfg = _lib.PriorConfig()
    cfg.width, cfg.depth, cfg.heads, cfg.n_state, cfg.mlp_width = W, 1, H, W // 4, W
    cfg.n_ctx, cfg.blocks, cfg.bins, cfg.prime_len, cfg.encoder_dims = n_ctx, blocks, 0, prime, enc
    cfg.max_batch, cfg.add_cond_after = max_batch, 1
    cfg.attn_func[0] = afs[-1]
    info = _lib.PlanInfo()
    _lib.check(_lib.lib().jk_prior_plan(C.byref(cfg), sms, C.byref(info), None, 0))
    return info.tile_rows


@pytest.mark.parametrize("name, max_batch", [("1b", 32), ("5b", 16), ("up", 32), ("many", 32), ("1b", 16)])
def test_tile_rows_match_plan(name, max_batch):
    g = geom(name)
    start = da.attn_tile_rows(g.dhp)
    assert plan_tile_rows(name, max_batch) == g.RC
    assert g.RC in [start >> k for k in range(4)]


def test_items_and_prefetch():
    g = geom("many")
    its = da.items(g, 32, 1, 100)
    assert len(its) == 512 and sum(i["prefetched"] for i in its) == 132
    assert [(i["b"], i["h"], i["s"]) for i in its[:3]] == [(0, 0, 0), (0, 1, 0), (0, 2, 0)]
    g = geom("1b")
    its = da.items(g, 16, 4, 500)
    assert len(its) == 128 and all(i["prefetched"] for i in its)
    assert [(i["b"], i["h"], i["s"]) for i in its[5:9]] == [(0, 1, 1), (0, 1, 2), (0, 1, 3), (1, 0, 0)]
    assert da.items(g, 16, 4, 0)[0]["prefetched"] is False


def test_div_small_and_partition():
    for d in (1, 2, 3, 4):
        for x in list(range(0, 2000)) + [98303]:
            assert da.div_small(x, d) == x // d
    g = geom("1b")
    for nc in range(0, 600):
        for ns in (1, 2, 3, 4):
            parts = da.partition(g, nc, ns, 1)
            rows = [r for pt in parts for r0, nr, _ in pt["tiles"] for r in range(r0, r0 + nr)]
            assert rows == list(range(nc))
            assert sum(c for pt in parts for _, _, c in pt["tiles"]) == 1


@pytest.mark.parametrize("dh, n, heads", [(16, 5, 1), (24, 40, 2), (64, 130, 4)])
def test_attend64_matches_attend_one(dh, n, heads):
    rng = np.random.default_rng(dh + n)
    S = dh * heads
    q = (2 * rng.standard_normal((1, S))).astype(np.float16)
    K = rng.standard_normal((1, n, S)).astype(np.float16)
    V = rng.standard_normal((1, n, S)).astype(np.float16)
    ref = attend_one(q.astype(np.float32), K.astype(np.float32), V.astype(np.float32), heads)[0]
    for h in range(heads):
        sl = slice(h * dh, (h + 1) * dh)
        _, p, a = da.attend64(q[0, sl], K[0, :, sl], V[0, :, sl], da.attn_scale2(dh))
        # attend_one keeps q.k in fp32 (no fp16 rounding of the scores): equal to their fp16 rounding, ~1e-3 relative
        np.testing.assert_allclose(a, ref[sl], atol=4e-3 * np.abs(V).max())
        assert abs(p.sum() - 1) < 1e-12


# ---- the bound against the emulation ------------------------------------------------------------------------------
def rows(rng, n, dh, kind):
    """K, V rows (fp16) of one head: N(0, 1.33) like the probe layer's LayerNorm outputs, or adversarial"""
    K = (1.15 * rng.standard_normal((n, dh))).astype(np.float16)
    V = (1.15 * rng.standard_normal((n, dh))).astype(np.float16)
    if kind == "adversarial":
        # values at fp16 rounding edges, a few huge v, keys in clusters with nearly equal scores
        V[::7] = np.float16(2047.0)
        V[1::7] = np.float16(-0.000123)
        K[::3] = K[0]
        K[1::11] *= np.float16(-1)
    return K, V


def query(rng, K, dh, e, kind):
    q = 1.15 * rng.standard_normal(dh)
    if kind == "adversarial":
        q = 0.9 * K[len(K) // 2].astype(np.float64) + 0.3 * q
    return (2.0 ** e * q).astype(np.float16)


def cases(name, G=132):
    """(ncache, ns, cur) sets of one geometry that reach every split, several tiles per part and a full last tile"""
    g = geom(name, G)
    t = g.trows
    out = [(t - 1, 1, 1), (t, 1, 1), (t + 1, 2, 1), (2 * t, 2, 1), (2 * t + 1, 3, 1), (3 * t + 1, 4, 1),
           (4 * 3 * t, 4, 1), (4 * 3 * t + 5, 4, 1), (2 * 5 * t - 1, 2, 0), (20 * t, 1, 1)]
    return g, [(nc, ns, cur) for nc, ns, cur in out if nc < 8576]


def within_bound(g, q, K, V, parts, shift, mutate=None):
    b, a, _ = da.bound(q, K, V, g, parts)
    got = da.emulate(q, K, V, g, parts, qk_shift=shift, mutate=mutate).astype(np.float64)
    return np.max(np.abs(got - a) / b), got


@pytest.mark.parametrize("name", list(REAL))
def test_emulation_within_bound(name):
    g, cs = cases(name)
    rng = np.random.default_rng(len(name))
    worst = 0.0
    for nc, ns, cur in cs:
        parts = da.partition(g, nc, ns, cur)
        n = nc + cur
        for e in (-8, -2, 0, 2, 3):
            for kind in ("random", "adversarial"):
                K, V = rows(rng, n, g.dh, kind)
                q = query(rng, K, g.dh, e, kind)
                _, _, a = da.attend64(q, K, V, g.scale2)
                dim = int(np.argmax(np.abs(V.astype(np.float64) - a[None]).sum(0)))
                adv = np.sign(V[:, dim].astype(np.float64) - a[dim])
                for shift in (None, rng.uniform(-1, 1, n), adv, -adv):
                    r, _ = within_bound(g, q, K, V, parts, shift)
                    worst = max(worst, r)
                    assert r <= 1.0, (name, nc, ns, cur, e, kind, r)
    print(name, "worst err / bound", worst)
    assert worst > 0.05        # the bound is not vacuous: rounding alone reaches a visible share of it


def test_mutated_arithmetic_exceeds_bound():
    """a missing corr rescale, a merge without expf(m_q - M): each exceeds the bound at real geometry"""
    g = geom("1b")
    rng = np.random.default_rng(5)
    nc = 12 * g.trows + 7
    parts = da.partition(g, nc, 4, 1)
    assert all(len(p["tiles"]) >= 3 for p in parts)
    for mutate in ("no_corr", "merge_no_w"):
        caught = False
        for e in (0, 2, 3):
            K, V = rows(rng, nc + 1, g.dh, "random")
            # a key that rises through the part: later tiles raise the running maximum
            K[5 * g.trows] = (3 * K[5 * g.trows].astype(np.float32)).astype(np.float16)
            q = query(rng, K, g.dh, e, "random")
            r, _ = within_bound(g, q, K, V, parts, None, mutate)
            caught |= r > 1.0
        assert caught, mutate


def route_exact(g, B_pos_k, B_pos_v, p, jstar, e, mutate=None, cache=None):
    """the exact routing check: a query aligned with the key of position jstar must return v of jstar, bit for bit"""
    kind, pos, cur = cache.read(p)
    if kind == "zeros":
        return True
    K, V = B_pos_k[pos], B_pos_v[pos]
    q = (2.0 ** e * B_pos_k[jstar].astype(np.float64)).astype(np.float16)
    parts = da.partition(g, len(pos) - cur, 1 if len(pos) - cur < g.RC else 2, cur)
    got = da.emulate(q, K, V, g, parts, mutate=mutate)
    return np.array_equal(got, B_pos_v[jstar])


@pytest.mark.parametrize("mutate, af", [("base+1", 1), ("transpose_as_p", 2), ("prev_swap", 3),
                                        ("cur_wrong_tile", 0), ("base+1", 0), ("no_corr", 0)])
def test_mutations_break_exact_routing(mutate, af):
    """route a query to the first / last cached row and the current token: the unmutated emulation returns v of that
    row bit for bit at every probe, each mutation misses at least one"""
    g = da.Geom(heads=1, dh=64, n_ctx=384, blocks=4, RC=64)
    rng = np.random.default_rng(7)
    Kp = rng.standard_normal((g.n_ctx, g.dh)).astype(np.float16)
    Vp = rng.standard_normal((g.n_ctx, g.dh)).astype(np.float16)
    layout_mut = mutate if mutate in ("base+1", "transpose_as_p", "prev_swap") else None
    arith_mut = None if layout_mut else mutate
    results = {}
    for label, lm, am in (("clean", None, None), ("mutated", layout_mut, arith_mut)):
        cache = da.CacheRows(g, af, lm)
        ok = True
        for p in range(g.n_ctx):
            want_kind, want = da.expected_rows(g, af, p)
            if p in (95, 96, 150, 200, 250, 287, 300, 383) and want_kind == "rows":
                for jstar in (want[0], want[-1], want[len(want) // 2]):
                    ok &= bool(route_exact(g, Kp, Vp, p, jstar, 4, mutate=am, cache=cache))
            cache.write(p)
        results[label] = ok
    assert results["clean"]
    assert not results["mutated"], f"{mutate} passed the exact routing check"
