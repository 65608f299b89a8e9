"""The fp32 transformer path (csrc/f32_path.cu) against float64 at the geometry the priors run it at.

The tiny golden fixtures stop at width 192, head_dim 48 and 96 positions.  These tests run one layer through
jk_f32_forward at the shapes of the 1b_lyrics, 5b_lyrics and upsampler priors - head_dim 256 / 150 / 480, 8 192 and
8 576 keys, block_ctx 134 / 64, the padded prime length 448, 512 encoder rows, fp16-stored Conv1D weights - and compare
it with oracle/transformer_f64.layer_f64, the reference's operators restated in float64 (pinned on the CPU by
test_f32_reference_cpu.py).

Tolerance.  layer_f64 carries a first-order bound of the fp32 error through the layer (its docstring derives it): every
dot product of K terms adds its own rounding, every later operator passes it on through its derivative.
  * worst  gamma_K sum |terms| per dot product, absolute values propagated: holds for any summation order.  At K = 2 048
           it is wider than the distance between two neighbouring patterns, so it cannot be the yardstick on its own.
  * stat   3 u sqrt(K) (||terms||_2 + |result|) per dot product, root-sum-square propagation: five standard deviations
           of the error of f32_path.cu's fma chains (u times each partial sum, independent signs).
Both are asserted (err / bound <= 1), on the layer's output and on the recorded attention weights (which must also be
exact zeros outside the pattern).  Sensitivity: every case evaluates the float64 layer a second time with its key set
shifted by one row (one block for the previous-block pattern).  The kernel must be at least 10 x the stat bound away
from that wrong answer in its attention weights (some key of some head) at every probe, and in its output at one probe
of the case at least.  The file runs in about 85 s on an H100 SXM.
The output alone cannot carry the check at every probe: one key more or less among hundreds or thousands moves the
layer's output by about that key's weight times a value row, which can sit within a few bounds (at 8 575 dense keys,
below one); the weights, compared key by key, tell the two patterns apart everywhere.  The printed margins show both.

The whole stack is compared with the reference's own fp32 outputs `y32` of
tests/golden/full*.npz at the fp32 path's contract of 2e-5.

Every number is printed, one JSON line per case (pytest -s)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err
from jukebox_b200 import _lib
from oracle.synth import synth_tensor
from oracle.transformer_f64 import attended_keys, layer_f64, layer_norm_bound
from oracle.transformer_np import prime_len_padded

pytestmark = pytest.mark.gpu

TOL32 = 2e-5
MARGIN = 10.0
CHUNK = 512

# (width, heads, n_ctx, blocks, prime_len, encoder_dims, fp16 Conv1D weights): the cfg of tests/golden/full*.npz
GEOM = {"1b": (2048, 2, 8576, 64, 384, 0, False),          # full1b_o12 / full1b_o9
        "5b": (4800, 8, 8192, 128, None, 512, True),        # full5b_o6
        "up": (1920, 1, 8192, 128, None, 0, False)}         # fullup_o2
CASES = [(0, "1b"), (1, "1b"), (1, "5b"), (1, "up"), (2, "1b"), (2, "5b"), (2, "up"),
         (3, "1b"), (3, "5b"), (3, "up"), (6, "5b"), (7, "1b")]


def record(row):
    print(json.dumps(row))


class Layer:
    """one layer of synthetic weights (oracle.synth, the reference's state-dict names) in a one-entry F32Layer table"""

    def __init__(self, width, heads, n_ctx, blocks, prime_len, encoder_dims, fp16, af, n_state=None, mlp=None, seed=5):
        self.W, self.H, self.n_ctx, self.blocks, self.prime_len = width, heads, n_ctx, blocks, prime_len
        self.S = n_state or width // 4
        self.Mw = mlp or width
        self.af, self.enc_dims = af, (encoder_dims if af == 6 else 0)
        self.bc = n_ctx // blocks
        self.prime = prime_len_padded(prime_len, blocks) if prime_len else None
        W, S, Mw = self.W, self.S, self.Mw
        shapes = [("ln_0.weight", (W,)), ("ln_0.bias", (W,)), ("attn.c_attn.w", (W, S if af == 6 else 3 * S)),
                  ("attn.c_attn.b", (S if af == 6 else 3 * S,)), ("attn.c_proj.w", (S, W)), ("attn.c_proj.b", (W,)),
                  ("ln_1.weight", (W,)), ("ln_1.bias", (W,)), ("mlp.c_fc.w", (W, Mw)), ("mlp.c_fc.b", (Mw,)),
                  ("mlp.c_proj.w", (Mw, W)), ("mlp.c_proj.b", (W,))]
        if af == 6:
            shapes += [("attn.c_enc_kv.w", (W, 2 * S)), ("attn.c_enc_kv.b", (2 * S,))]
        self.p32 = {}
        for name, shape in shapes:
            a = synth_tensor(f"_attn_mods.0.{name}", shape, seed)
            if fp16 and name.endswith(".w"):        # make_models.py stores Conv1D weights in fp16; the path widens them
                a = a.astype(np.float16).astype(np.float32)
            self.p32[name] = torch.from_numpy(a).cuda()
        self.p64 = {k: v.double() for k, v in self.p32.items()}
        L = _lib.F32Layer()
        p = self.p32
        for field, name in (("ln0_g", "ln_0.weight"), ("ln0_b", "ln_0.bias"), ("ln1_g", "ln_1.weight"),
                            ("ln1_b", "ln_1.bias"), ("c_attn_w", "attn.c_attn.w"), ("c_attn_b", "attn.c_attn.b"),
                            ("c_proj_w", "attn.c_proj.w"), ("c_proj_b", "attn.c_proj.b"), ("fc_w", "mlp.c_fc.w"),
                            ("fc_b", "mlp.c_fc.b"), ("proj2_w", "mlp.c_proj.w"), ("proj2_b", "mlp.c_proj.b")):
            setattr(L, field, p[name].data_ptr())
        if af == 6:
            L.c_enc_kv_w, L.c_enc_kv_b = p["attn.c_enc_kv.w"].data_ptr(), p["attn.c_enc_kv.b"].data_ptr()
        L.attn_func = af
        self.L = L
        self.work = None

    def caches(self, n, fill=float("nan")):
        """fresh K/V caches; NaN rows show any row read before it was written, and any row never written"""
        rows = self.enc_dims if self.af == 6 else self.n_ctx
        self.kc = torch.full((n, rows, self.S), fill, device="cuda")
        self.vc = torch.full((n, rows, self.S), fill, device="cuda")
        self.L.k_cache, self.L.v_cache = self.kc.data_ptr(), self.vc.data_ptr()

    def args(self, x, p0, enc=None, depth=1):
        n, P, _ = x.shape
        return _lib.F32Args(n=n, P=P, p0=p0, width=self.W, n_state=self.S, mlp_width=self.Mw, heads=self.H,
                            n_ctx=self.n_ctx, blocks=self.blocks, prime_len=self.prime_len or 0,
                            encoder_dims=self.enc_dims, depth=depth, x=x.data_ptr(),
                            encoder_kv=0 if enc is None else enc.data_ptr(), work=0)

    def run(self, x, p0, enc=None, record_w=False):
        """x [n, P, width] fp32 through the layer at positions [p0, p0 + P) (in place); returns the weights if asked"""
        n, P, _ = x.shape
        a = self.args(x, p0, enc)
        need = C.c_size_t(0)
        _lib.check(_lib.lib().jk_f32_workspace_floats(C.byref(a), C.byref(need)))
        if self.work is None or self.work.numel() < need.value:
            self.work = torch.empty(need.value, device="cuda")
        a.work = self.work.data_ptr()
        w = None
        if record_w:
            w = torch.full((n, self.H, P, self.enc_dims if self.af == 6 else self.n_ctx), float("nan"), device="cuda")
            self.L.attn_w = w.data_ptr()
        else:
            self.L.attn_w = 0
        _lib.check(_lib.lib().jk_f32_forward(C.byref(a), C.pointer(self.L), _lib.stream_ptr()))
        self.L.attn_w = 0
        return w

    def f64(self, x64, queries, enc64=None, shift=0, bound=None):
        return layer_f64(self.p64, x64, queries, self.af, self.H, self.bc, self.prime, enc64, shift, bound)


def geom_layer(af, g):
    W, H, n_ctx, blocks, prime_len, enc, fp16 = GEOM[g]
    return Layer(W, H, n_ctx, blocks, prime_len, enc, fp16, af)


def inputs(ly, n, seed):
    """residual-stream rows of the fixtures' magnitude (|h| up to ~25): N(0, 2^2) plus a per-row offset"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = 2.0 * torch.randn(n, ly.n_ctx, ly.W, device="cuda", generator=gen)
    x += torch.randn(n, ly.n_ctx, 1, device="cuda", generator=gen)
    enc = None
    if ly.af == 6:
        enc = 2.0 * torch.randn(n, ly.enc_dims, ly.W, device="cuda", generator=gen)
    return x, enc


def probes(ly):
    bc, p = ly.bc, [0, 1, ly.bc - 1, ly.bc, ly.bc + 1, 2 * ly.bc - 1, 2 * ly.bc]
    if ly.af == 7:
        p += [ly.prime - 1, ly.prime, ly.prime + 1]
    return sorted(set(p + [4000, ly.n_ctx - 1]))


def compare(ly, y, w, x64, qs, enc64):
    """kernel rows y [n, Q, W] and recorded weights w [n, H, Q, keys] at positions qs against float64.  Returns the
    worst / stat ratios of y, the stat ratio of w inside the pattern, the largest |w| outside it, and the sensitivity
    margins per probe - (keys, margin of y, margin of w), skipped where the shifted key set is the same set."""
    st = ly.f64(x64, qs, enc64, bound="stat")
    wc = ly.f64(x64, qs, enc64, bound="worst")
    err = (y.double() - st["y"]).abs()
    r_stat = float((err / st["ey"]).max())
    r_worst = float((err / wc["ey"]).max())
    w = w.double()
    inside = st["w"] != 0
    werr = float(((w - st["w"]).abs() / st["ew"]).where(inside, torch.zeros_like(w)).max())
    outside = float(w.where(~inside, torch.zeros_like(w)).abs().max())
    shift = ly.bc if ly.af == 3 else 1
    wrong = ly.f64(x64, qs, enc64, shift=shift)
    dist_y = (y.double() - wrong["y"]).abs() / st["ey"]
    # a weight the right pattern leaves at 0 has no error of its own: measure the distance there in units of the
    # bound of the largest weight of the row (of one rounding of a weight of 1 in the zero block)
    wtol = torch.where(inside, st["ew"], st["ew"].amax(-1, keepdim=True)).clamp_min(2.0 ** -24)
    dist_w = (w - wrong["w"]).abs() / wtol
    margins = []
    n_keys = ly.enc_dims if ly.af == 6 else ly.n_ctx
    for i, p in enumerate(qs):
        a = attended_keys(ly.af, p, ly.bc, ly.prime, n_keys)
        b = attended_keys(ly.af, p, ly.bc, ly.prime, n_keys, shift)
        if (a is None and b is None) or (a is not None and b is not None and np.array_equal(a, b)):
            continue
        nk = 0 if a is None else len(a)
        # per sample: the largest distance over the row (over every head and key for the weights)
        margins.append((nk, float(dist_y[:, i].amax(-1).min()), float(dist_w[:, :, i].amax((1, 2)).min())))
    return dict(err_over_stat_bound=round(r_stat, 4), err_over_worst_bound=float(f"{r_worst:.3e}"),
                weights_err_over_stat_bound=round(werr, 4), weights_outside_pattern=outside,
                wrong_pattern_margin_y=[round(m[1], 1) for m in margins],
                wrong_pattern_margin_w=[float(f"{m[2]:.3g}") for m in margins]), margins, st


def check(row, margins):
    assert row["err_over_stat_bound"] <= 1.0 and row["err_over_worst_bound"] <= 1.0, row
    assert row["weights_err_over_stat_bound"] <= 1.0 and row["weights_outside_pattern"] == 0.0, row
    assert min(m[2] for m in margins) >= MARGIN, margins
    assert max(m[1] for m in margins) >= MARGIN, margins


@pytest.mark.parametrize("af, g", CASES)
def test_one_layer_forward_mode_against_float64(af, g):
    """p0 = 0, P = n_ctx: the whole window in one call, compared at the probes; recorded attention weights too"""
    ly = geom_layer(af, g)
    n = 2
    x, enc = inputs(ly, n, 100 + af)
    x64, enc64 = x.double(), None if enc is None else enc.double()
    qs = probes(ly)
    ly.caches(n)
    y = x.clone()
    w = ly.run(y, 0, enc, record_w=True)
    torch.cuda.synchronize()
    yq = y[:, qs]
    wq = w[:, :, qs]
    del w
    row, margins, _ = compare(ly, yq, wq, x64, qs, enc64)
    record(dict(case=f"forward af{af} {g}", dh=ly.S // ly.H, n_ctx=ly.n_ctx, block_ctx=ly.bc, probes=qs, **row))
    assert torch.isfinite(yq).all()
    check(row, margins)
    if af == 3:
        first = [i for i, p in enumerate(qs) if p < ly.bc]
        assert float(wq[:, :, first].abs().max()) == 0.0


def sampling_probes(ly):
    """the probes of sampling mode: the prime boundary's own probes give way to one chunk that crosses it"""
    qs = probes(ly)
    if ly.af == 7:
        qs = [p for p in qs if p not in (ly.prime - 1, ly.prime)]
    return qs


@pytest.mark.parametrize("af, g", CASES)
def test_one_layer_sampling_mode_against_float64(af, g):
    """caches primed in chunks that end just before each probe (chunks of up to 512 cross block boundaries; for the
    prime layer one crosses _prime_len), then the probe alone (P = 1): output, and the K / V row it wrote"""
    ly = geom_layer(af, g)
    n = 2
    x, enc = inputs(ly, n, 200 + af)
    x64, enc64 = x.double(), None if enc is None else enc.double()
    qs = sampling_probes(ly)
    ly.caches(n)
    ys, ws, cur, crossed_block, crossed_prime = [], [], 0, False, False
    for p in qs:
        while cur < p:
            c = min(CHUNK, p - cur)
            crossed_block |= (cur // ly.bc) != ((cur + c - 1) // ly.bc)
            crossed_prime |= ly.prime is not None and cur < ly.prime <= cur + c - 1
            ly.run(x[:, cur:cur + c].clone(), cur, enc if cur == 0 else None)
            cur += c
        y = x[:, p:p + 1].clone()
        ws.append(ly.run(y, p, enc if p == 0 else None, record_w=True)[:, :, 0])
        ys.append(y[:, 0])
        cur = p + 1
    torch.cuda.synchronize()
    assert crossed_block and (af != 7 or crossed_prime)
    yq = torch.stack(ys, 1)
    row, margins, st = compare(ly, yq, torch.stack(ws, 2), x64, qs, enc64)
    # the cache rows of the probes (absolute positions), against the float64 K / V
    if af == 6:
        rows = list(range(ly.enc_dims))
    else:
        rows = [p for p in qs if af != 7 or p < ly.prime]
    kv_ratio = 0.0
    for got, want, bound in ((ly.kc, st["k"], st["ek"]), (ly.vc, st["v"], st["ev"])):
        e = (got[:, rows].double() - want[:, rows]).abs() / bound[:, rows]
        kv_ratio = max(kv_ratio, float(e.max()))
    unwritten_ok = True
    if af == 7:      # prime layer: rows at and past _prime_len are never written
        unwritten_ok = bool(torch.isnan(ly.kc[:, ly.prime:]).all() and torch.isnan(ly.vc[:, ly.prime:]).all())
        assert bool(torch.isfinite(ly.kc[:, :ly.prime]).all())
    record(dict(case=f"sampling af{af} {g}", probes=qs, kv_rows_err_over_stat_bound=round(kv_ratio, 4),
                prime_rows_unwritten=unwritten_ok, **row))
    assert torch.isfinite(yq).all()
    check(row, margins)
    assert kv_ratio <= 1.0 and unwritten_ok


# ---- GEMM epilogues and tile edges: partial 64 x 64 tiles, K tails of the 16-deep loop, GELU, residual in place ----
@pytest.mark.parametrize("W, S, Mw, H", [(72, 36, 200, 2), (130, 65, 390, 5)])
@pytest.mark.parametrize("n, P", [(1, 1), (1, 63), (1, 64), (1, 65), (3, 43)])
def test_small_odd_layer_tile_edges(W, S, Mw, H, n, P):
    ly = Layer(W, H, 160, 4, None, 0, False, 1, n_state=S, mlp=Mw, seed=W + P)
    x, _ = inputs(ly, n, W * 1000 + P)
    ly.caches(n)
    y = x[:, :P].clone()
    ly.run(y, 0)
    qs = list(range(P))
    x64 = x[:, :P].double()
    st = ly.f64(x64, qs, bound="stat")
    wc = ly.f64(x64, qs, bound="worst")
    err = (y.double() - st["y"]).abs()
    r_stat, r_worst = float((err / st["ey"]).max()), float((err / wc["ey"]).max())
    record(dict(case=f"tile edges W {W} S {S} mlp {Mw} rows {n * P}", err_over_stat_bound=round(r_stat, 4),
                err_over_worst_bound=float(f"{r_worst:.3e}")))
    assert r_stat <= 1.0 and r_worst <= 1.0


# ---- the whole stack against the reference's fp32 outputs at baseline geometry ----------------------------------
@pytest.mark.parametrize("tag", ["full1b_o12", "full1b_o9", "full5b_o6", "fullup_o2"])
def test_stack_matches_reference_fp32(tag):
    from test_gpu_fullsize_golden import build
    fx = Fixture(tag)
    c = fx.cfg
    tr = build(fx)          # fp16_params: Conv1D weights stored in fp16, widened by the fp32 path
    x = torch.from_numpy(synth_tensor("input.x", (c["bs"], c["n_ctx"], c["n_in"]), c["seed"])).cuda()
    enc = None
    if c["encoder_dims"]:
        enc = torch.from_numpy(synth_tensor("input.encoder_kv", (c["bs"], c["encoder_dims"], c["n_in"]), c["seed"])).cuda()
    qs = c["probes"]
    ys = []
    with torch.no_grad():
        tr.del_cache()
        cur = 0
        for p in qs:             # as oracle/make_golden_fullsize.py drove the reference
            while cur < p:
                k = min(c["chunk"], p - cur)
                tr(x[:, cur:cur + k].contiguous(), encoder_kv=enc, sample=True, fp16=False)
                cur += k
            ys.append(tr(x[:, p:p + 1].contiguous(), encoder_kv=enc, sample=True, fp16=False)[:, 0])
            cur = p + 1
        tr.del_cache()
        y_samp = torch.stack(ys, 1).cpu().numpy()
        y_fwd = tr(x, encoder_kv=enc, sample=False, fp16=False)[:, qs].cpu().numpy()
    y32 = fx["y32"]
    es, ef = rel_err(y_samp, y32), rel_err(y_fwd, y32)
    record(dict(fixture=tag, api="Transformer.forward(fp16=False)", sampling_vs_ref_fp32=es, forward_vs_ref_fp32=ef,
                sampling_vs_forward=rel_err(y_samp, y_fwd), max_abs_ref=float(np.abs(y32).max()), tol=TOL32))
    assert np.isfinite(y_samp).all() and np.isfinite(y_fwd).all()
    assert es <= TOL32 and ef <= TOL32


# ---- argument errors are returned before any launch -------------------------------------------------------------
def _forward_rc(layers, a):
    table = (_lib.F32Layer * len(layers))(*layers)
    need = C.c_size_t(0)
    _lib.check(_lib.lib().jk_f32_workspace_floats(C.byref(a), C.byref(need)))
    work = torch.empty(need.value, device="cuda")
    a.work = work.data_ptr()
    rc = _lib.lib().jk_f32_forward(C.byref(a), table, _lib.stream_ptr())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("bad", ["attn_func 4", "no cache", "shared memory"])
def test_invalid_layer_table_leaves_x_unchanged(bad):
    """a table whose last layer cannot run is refused before layer 0 touches x"""
    n = 1
    if bad == "shared memory":
        # layer 0: encoder-decoder over 8 rows (fits); layer 1: a block layer whose attention row would hold
        # n_ctx + head_dim floats, past the 96 KB the kernel is given
        l0 = Layer(72, 2, 24576, 4, None, 8, False, 6, n_state=36, mlp=200, seed=1)
        l1 = Layer(72, 2, 24576, 4, None, 0, False, 1, n_state=36, mlp=200, seed=2)
    else:
        l0 = Layer(72, 2, 160, 4, None, 0, False, 1, n_state=36, mlp=200, seed=1)
        l1 = Layer(72, 2, 160, 4, None, 0, False, 2, n_state=36, mlp=200, seed=2)
    l2 = Layer(72, 2, l0.n_ctx, 4, None, 0, False, 3, n_state=36, mlp=200, seed=3)
    for ly in (l0, l1, l2):
        ly.caches(n, 0.0)
    enc = torch.randn(n, 8, 72, device="cuda") if l0.af == 6 else None
    x = torch.randn(n, 5, 72, device="cuda")
    before = x.clone()
    good = [l0.L, l1.L, l2.L]
    bad_l = _lib.F32Layer.from_buffer_copy(l2.L)
    if bad == "attn_func 4":
        bad_l.attn_func = 4
    elif bad == "no cache":
        bad_l.v_cache = 0
    layers = [l0.L, l1.L] if bad == "shared memory" else [l0.L, l1.L, bad_l]
    a = l0.args(x, 0, enc, depth=len(layers))
    a.encoder_dims = 8 if bad == "shared memory" else 0
    rc = _forward_rc(layers, a)
    err = _lib.lib().jk_last_error().decode()
    print(f"{bad}: rc {rc}: {err}")
    assert rc != 0
    assert torch.equal(x.view(torch.int32), before.view(torch.int32))
    if bad != "shared memory":        # the same call with a valid last layer does run
        a = l0.args(x, 0, None, depth=3)
        assert _forward_rc(good, a) == 0 and not torch.equal(x, before)


# ---- jk_layernorm_f32 (the Conditioner's LayerNorm and both LayerNorms of the fp32 path) --------------------------
@pytest.mark.parametrize("W", [1, 255, 257, 1920, 4800])
def test_layernorm_f32_against_float64(W):
    gen = torch.Generator(device="cuda").manual_seed(W)
    rows = [torch.randn(W, device="cuda", generator=gen) * 3,
            1e3 + 1e-2 * torch.randn(W, device="cuda", generator=gen),       # |mean| >> std
            -250.0 + 1e-3 * torch.randn(W, device="cuda", generator=gen),
            torch.full((W,), 0.1, device="cuda"), torch.full((W,), 1e3, device="cuda"),      # constant rows
            torch.zeros(W, device="cuda")]
    x = torch.stack(rows)
    g = 1.0 + 0.1 * torch.randn(W, device="cuda", generator=gen)
    b = 0.1 * torch.randn(W, device="cuda", generator=gen)
    y = torch.empty_like(x)
    _lib.check(_lib.lib().jk_layernorm_f32(_lib.ptr(x), _lib.ptr(g), _lib.ptr(b), _lib.ptr(y), x.shape[0], W, 1e-5,
                                           _lib.stream_ptr()))
    want, bound = layer_norm_bound(x.double(), None, g.double(), b.double())
    ratio = ((y.double() - want).abs() / bound).amax(-1)
    # one-pass statistics (E[x^2] - mean^2 in fp32) are what the large-mean rows would expose
    print(f"jk_layernorm_f32 W {W}: err / bound per row {[round(float(r), 4) for r in ratio]}")
    assert torch.isfinite(y).all()
    assert float(ratio.max()) <= 1.0


# ---- jk_f32_embed: (x_emb[token] or the position-0 row) + pos_emb, + x_cond, bit for bit ---------------------------
@pytest.mark.parametrize("start, xc_len, p0, P", [("y_cond", 0, 0, 40), ("start_token", 1, 0, 40),
                                                  ("y_cond", "n_ctx", 0, 40), ("start_token", "n_ctx", 0, 1),
                                                  ("y_cond", 1, 17, 23), ("start_token", "n_ctx", 33, 7),
                                                  ("y_cond", 0, 39, 1)])
def test_f32_embed_bit_exact(start, xc_len, p0, P):
    n, n_ctx, W, bins = 3, 40, 96, 50
    gen = torch.Generator(device="cuda").manual_seed(p0 * 100 + P)
    emb = torch.randn(bins, W, device="cuda", generator=gen)
    pos = torch.randn(n_ctx, W, device="cuda", generator=gen) * 0.5
    st = torch.randn(W, device="cuda", generator=gen)
    yc = torch.randn(n, W, device="cuda", generator=gen)
    L = n_ctx if xc_len == "n_ctx" else xc_len
    xc = torch.randn(n, L, W, device="cuda", generator=gen) if L else None
    wide = torch.randint(0, bins, (n, n_ctx + 9), device="cuda", generator=gen)
    tokens = wide[:, 3:3 + n_ctx]                      # a strided view: row stride n_ctx + 9
    assert tokens.stride(0) == n_ctx + 9
    tok_ptr = C.c_void_p(wide.data_ptr() + 3 * wide.element_size())
    out = torch.full((n, P, W), float("nan"), device="cuda")
    _lib.check(_lib.lib().jk_f32_embed(_lib.ptr(out), tok_ptr, tokens.stride(0),
                                       _lib.ptr(yc if start == "y_cond" else None), _lib.ptr(xc), L,
                                       _lib.ptr(emb), _lib.ptr(pos), _lib.ptr(st if start == "start_token" else None),
                                       n, P, p0, W, _lib.stream_ptr()))
    want = torch.empty(n, P, W, device="cuda")
    for i in range(P):
        t = p0 + i
        if t == 0:
            first = yc if start == "y_cond" else st.expand(n, W)
        else:
            first = emb[tokens[:, t - 1]]
        v = first + pos[t]
        if xc is not None:
            v = v + (xc[:, t] if L > 1 else xc[:, 0])
        want[:, i] = v
    assert torch.equal(out.view(torch.int32), want.view(torch.int32))
