"""Representations from a prior's intermediate layers on the GPU: the truncated fp16 prefill with in-pass layer capture and
pooling (jk_prefill_args.n_layers / capture, csrc/prefill.cu act_rows_kernel), the fp32 route (F32Path.run_layers +
jk_pool_rows_f32), and the Python surface (ConditionalAutoregressive2D / SimplePrior.layer_acts).

  reference  - layer_acts against the reference's JukeMIR recipe (tests/golden/acts_*.npz): fp16 within 5e-3 of the
               reference's fp16 pass (the prefill tests' bound), fp32 within 2e-5 of its fp32 pass (the fp32 path's bound)
  bits       - a capture at depth-1 of an n_layers = depth call is h_out; a capture at L of an n_layers = L+1 call is the
               capture at L of a full call; the new fields left at zero change no output of the prefill or the steps
  pooling    - the mean equals the mean of the rows; its bits do not depend on the batch or the run; both routes pool
               through the same kernel
  state      - after a truncated prefill the engine refuses to step or prefill until reset, then samples as a fresh one
  errors     - every invalid capture is an error with a message, and nothing is written
  5b         - prior_5b geometry, 2 items x 8192 positions, layer 36: finite, and the fp16 / fp32 difference is reported"""
import pytest
import torch

from golden_util import Fixture, rel_err
from test_gpu_prefill import _model
from test_gpu_prior import _make_prior

pytestmark = pytest.mark.gpu

TAGS = ["labelled", "single_enc_dec", "sep_enc_dec"]


@pytest.mark.parametrize("tag", TAGS)
def test_layer_acts_match_the_reference(tag):
    fx = Fixture(f"acts_{tag}")
    prior = _make_prior(fx)
    layers = fx.cfg["layers"]
    z, y = torch.from_numpy(fx["z"]).cuda(), torch.from_numpy(fx["y"]).cuda()
    tr = prior.prior.transformer
    for fp16, key, tol in ((True, "a16", 5e-3), (False, "a32", 2e-5)):
        rows = prior.layer_acts(z, [], y, layers=layers, fp16=fp16, pool=False)
        pooled = prior.layer_acts(z, [], y, layers=layers, fp16=fp16, pool=True)
        for l in layers:
            ref = fx[f"{key}_{l}"]
            assert rows[l].shape == ref.shape and pooled[l].shape == (ref.shape[0], ref.shape[2])
            e, ep = rel_err(rows[l].cpu().numpy(), ref), rel_err(pooled[l].cpu().numpy(), ref.mean(1))
            print(f"acts_{tag} layer {l} fp16={fp16}: rows {e:.2e}, pooled {ep:.2e} (bound {tol:g})")
            assert e < tol and ep < tol
        if fp16:
            assert tr._f32 is None, "the fp16 route must not build the fp32 path"
            assert tr._engine.position == 0, "layer_acts leaves the engine reset"


def _tiny(seed=3, x_cond=True):
    m, _ = _model(2, 256, 6, 2, 128, 4, seed=seed, x_cond=x_cond)
    return m


def _inputs(m, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randint(0, m.bins, (n, m.input_dims), generator=g).cuda()
    yc = torch.randn(n, m.width, generator=g).cuda()
    xc = torch.randn(n, m.input_dims, m.width, generator=g).cuda() * 0.1 if m.x_cond else None
    return tokens, yc, xc


def _prefill(m, n, P, tokens, yc, xc, **kw):
    from jukebox_b200.engine import Capture
    tr = m.transformer
    tr.del_cache()
    eng = m._engine(n)
    cap = {l: Capture(*c) for l, c in kw.pop("capture", {}).items()}
    eng.prefill(n, P, tokens=tokens, y_cond=yc, x_cond=xc, capture=cap, **kw)
    torch.cuda.synchronize()
    return eng


def test_truncated_capture_is_the_full_prefill_bit_for_bit():
    m = _tiny()
    n, P, W, depth = 3, 100, m.width, m.depth
    tokens, yc, xc = _inputs(m, n)
    h = torch.empty(n, P, W, device="cuda")
    _prefill(m, n, P, tokens, yc, xc, h_out=h)
    last = torch.empty(n, P, W, device="cuda")
    _prefill(m, n, P, tokens, yc, xc, n_layers=depth, capture={depth - 1: (last, 0, P, False, False)})
    assert torch.equal(last, h)
    full = {l: torch.empty(n, P, W, device="cuda") for l in range(depth)}
    _prefill(m, n, P, tokens, yc, xc, capture={l: (b, 0, P, False, False) for l, b in full.items()})
    for L in (0, 2, 4):
        cut, hcut = torch.empty(n, P, W, device="cuda"), torch.empty(n, P, W, device="cuda")
        eng = _prefill(m, n, P, tokens, yc, xc, n_layers=L + 1, h_out=hcut, capture={L: (cut, 0, P, False, False)})
        assert eng.position == -1
        assert torch.equal(cut, full[L]) and torch.equal(hcut, full[L]), L
        pooled = torch.empty(n, W, device="cuda")
        _prefill(m, n, P, tokens, yc, xc, n_layers=L + 1, capture={L: (pooled, 0, P, True, False)})
        assert torch.allclose(pooled.double(), full[L].double().mean(1), rtol=0, atol=1e-6 * float(full[L].abs().max()))
    m.transformer.del_cache()


def test_new_fields_at_zero_change_no_output():
    from jukebox_b200.transformer.ops import sample_categorical
    m = _tiny()
    tr = m.transformer
    n, P, K = 2, 64, 6
    tokens, yc, xc = _inputs(m, n, seed=1)
    results = []
    for kw in ({}, dict(n_layers=0, capture={}), dict(n_layers=m.depth, capture={1: (torch.empty(n, m.width, device="cuda"), 3, 50, True, True)})):
        h = torch.empty(n, P, m.width, device="cuda")
        ws = {i: torch.empty(n, tr.n_head, P, P, dtype=torch.float16, device="cuda") for i in (0, 3)}
        eng = _prefill(m, n, P, tokens, yc, xc, h_out=h, record=ws, **kw)
        assert eng.position == P
        lbuf = torch.empty(n, m.bins, device="cuda")
        toks = tokens.clone()
        logits = []
        for k in range(K):
            eng.step(n, tokens=toks, y_cond=yc, x_cond=xc, logits=lbuf)
            logits.append(lbuf.clone())
            sample_categorical(lbuf, 1.0, 77, P + k, toks)
        results.append((h, ws, torch.stack(logits), toks))
    for h, ws, lg, tk in results[1:]:
        assert torch.equal(h, results[0][0]) and torch.equal(lg, results[0][2]) and torch.equal(tk, results[0][3])
        assert all(torch.equal(ws[i], results[0][1][i]) for i in ws)
    tr.del_cache()


def test_pooled_bits_do_not_depend_on_the_batch_or_the_run():
    m, _ = _model(2, 256, 4, 2, 128, 4, seed=5, x_cond=True)
    N, P = 32, 128
    tokens, yc, xc = _inputs(m, N, seed=2)
    m._engine(32)
    outs = {}
    for n in (1, 16, 32, 32):
        o = torch.empty(n, m.width, device="cuda")
        _prefill(m, n, P, tokens[:n].contiguous(), yc[:n].contiguous(), xc[:n].contiguous(), n_layers=3,
                 capture={2: (o, 5, P, True, True)})
        outs.setdefault(n, []).append(o)
    assert torch.equal(outs[16][0][0], outs[1][0][0]) and torch.equal(outs[32][0][:16], outs[16][0])
    assert torch.equal(outs[32][0], outs[32][1])
    # the fp16 route's mean is the mean of its rows (x_cond added), and the fp32 route pools with the same kernel
    rows = torch.empty(N, P - 5, m.width, device="cuda")
    _prefill(m, N, P, tokens, yc, xc, n_layers=3, capture={2: (rows, 5, P, False, True)})
    want = rows.double().mean(1)
    assert torch.allclose(outs[32][0].double(), want, rtol=0, atol=1e-6 * float(rows.abs().max()))
    from jukebox_b200 import _lib
    x_rows = torch.cat([torch.zeros(N, 5, m.width, device="cuda"), rows], 1).contiguous()
    p32 = torch.empty(N, m.width, device="cuda")
    _lib.check(_lib.lib().jk_pool_rows_f32(_lib.ptr(x_rows), N, P, m.width, 5, P, None, 0, _lib.ptr(p32), _lib.stream_ptr()))
    assert torch.equal(p32, outs[32][0]), "both routes pool through the same kernel"
    m.transformer.del_cache()


def test_a_truncated_engine_must_be_reset_then_samples_as_a_fresh_one():
    m = _tiny(x_cond=False)
    n, P = 2, 40
    tokens, yc, _ = _inputs(m, n, seed=4)
    eng = _prefill(m, n, P, tokens, yc, None, n_layers=2)
    assert eng.position == -1
    from jukebox_b200._lib import lib
    import ctypes
    t = ctypes.c_int(5)
    assert lib().jk_prior_position(eng.handle, ctypes.byref(t)) == 0 and t.value == -1
    with pytest.raises(RuntimeError, match="jk_prior_reset"):
        eng.step(n, tokens=tokens, y_cond=yc)
    with pytest.raises(RuntimeError, match="jk_prior_reset"):
        eng.prefill(n, P, tokens=tokens, y_cond=yc)
    prime = tokens[:, :30].clone()
    torch.manual_seed(11)
    after = m.primed_sample(n, prime, y_cond=yc[:, None], fp16=True, sample_tokens=50)       # resets the engine first
    m.transformer.drop_engine()
    torch.manual_seed(11)
    fresh = m.primed_sample(n, prime, y_cond=yc[:, None], fp16=True, sample_tokens=50)
    assert torch.equal(after, fresh)


def test_invalid_captures_are_errors_and_write_nothing():
    from jukebox_b200.engine import Capture
    m = _tiny()
    n, P, W = 2, 64, m.width
    tokens, yc, xc = _inputs(m, n, seed=6)
    eng = m._engine(n)
    m.transformer.del_cache()
    out = torch.full((n, W), 7.0, device="cuda")
    h = torch.full((n, P, W), 7.0, device="cuda")
    bad = [
        (dict(capture={m.depth: Capture(out, 0, P, True, False)}), "out of range"),
        (dict(capture={-1: Capture(out, 0, P, True, False)}), "out of range"),
        (dict(n_layers=3, capture={3: Capture(out, 0, P, True, False)}), "out of range"),
        (dict(capture={2: Capture(out, 5, 5, True, False)}), "empty or outside"),
        (dict(capture={2: Capture(out, 10, P + 1, True, False)}), "empty or outside"),
        (dict(capture={2: Capture(out, -1, 4, True, False)}), "empty or outside"),
        (dict(x_cond=None, capture={2: Capture(out, 0, P, True, True)}), "adds x_cond"),
        (dict(n_layers=m.depth + 1), "n_layers"),
    ]
    for kw, msg in bad:
        args = dict(tokens=tokens, y_cond=yc, x_cond=xc, h_out=h)
        args.update(kw)
        with pytest.raises(RuntimeError, match=msg):
            eng.prefill(n, P, **args)
        assert eng.position == 0 or eng.position == P      # the Python mirror is only updated on success
    # a layer listed twice and a NULL output go through the C table directly
    import ctypes
    from jukebox_b200 import _lib
    for entries, msg in (([(2, out), (2, out)], "listed twice"), ([(2, None)], "no output buffer")):
        a = _lib.PrefillArgs()
        a.n_samples, a.n_positions, a.tokens, a.tok_stride = n, P, _lib.ptr(tokens), tokens.stride(0)
        a.y_cond, a.x_cond, a.x_cond_len, a.h_out = _lib.ptr(yc), _lib.ptr(xc), xc.shape[1], _lib.ptr(h)
        table = (_lib.ActCapture * len(entries))()
        for e, (l, o) in zip(table, entries):
            e.layer, e.t0, e.t1, e.pool, e.out = l, 0, P, 1, _lib.ptr(o)
        a.capture, a.n_capture = table, len(entries)
        assert _lib.lib().jk_prior_prefill(eng.handle, ctypes.byref(a), _lib.stream_ptr()) != 0
        assert msg.encode() in _lib.lib().jk_last_error()
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()) and bool((h == 7.0).all()), "a refused call wrote its outputs"
    t = ctypes.c_int(9)
    _lib.lib().jk_prior_position(eng.handle, ctypes.byref(t))
    assert t.value == 0, "a refused call moved the engine"


def test_short_windows_are_the_full_window_prefix():
    m = _tiny()
    n = 2
    tokens, yc, xc = _inputs(m, n, seed=8)
    full = m.layer_acts(tokens, xc, yc[:, None], layers=(1, 4), pool=False)
    for fp16 in (True, False):
        short = m.layer_acts(tokens[:, :70], xc, yc[:, None], layers=(1, 4), pool=False, fp16=fp16)
        ref = full if fp16 else m.layer_acts(tokens, xc, yc[:, None], layers=(1, 4), pool=False, fp16=False)
        for l in (1, 4):
            assert torch.equal(short[l], ref[l][:, :70]) if fp16 else \
                torch.allclose(short[l], ref[l][:, :70], rtol=0, atol=2e-5 * float(ref[l].abs().max()))


def test_prior_5b_geometry_layer_36():
    """2 items x 8192 positions of prior_5b geometry (width 4800, 8 heads, attn_order 2, blocks 128, label-conditioned) with
    synthetic weights, layer 36 pooled.  The stack is cut after layer 37: a 72-layer model computes the same layer 36, the
    prefix (tools/acts_time.py runs all 72).  The fp16 / fp32 gap is reported; the bound is the reference fixtures' gap,
    which grows with depth: ref16 vs ref32 reaches 2.3e-3 of the row range after 16 layers, so 36 layers of width 4800 are
    allowed 2e-2 of the pooled range."""
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = ConditionalAutoregressive2D((8192,), 2048, width=4800, depth=37, heads=8, attn_order=2, blocks=128,
                                        init_scale=0.1, x_cond=True, y_cond=True, merged_decoder=True).eval()
    n = 2
    g = torch.Generator(device="cuda").manual_seed(1)
    tokens = torch.randint(0, 2048, (n, 8192), device="cuda", generator=g)
    yc = torch.randn(n, 1, 4800, device="cuda", generator=g) * 0.1
    xc = torch.randn(n, 8192, 4800, device="cuda", generator=g) * 0.01
    f16 = m.layer_acts(tokens, xc, yc, layers=(36,), fp16=True)[36]
    m.transformer.drop_engine()
    torch.cuda.empty_cache()
    f32 = m.layer_acts(tokens, xc, yc, layers=(36,), fp16=False)[36]
    assert torch.isfinite(f16).all() and torch.isfinite(f32).all()
    e = rel_err(f16.cpu().numpy(), f32.cpu().numpy())
    print(f"prior_5b geometry, layer 36, 2 x 8192: max|fp16 - fp32| / max|fp32| of the pooled features {e:.2e}")
    assert e < 2e-2
