"""Sample selection on the GPU (jk_prior_select, csrc/select.cu).

Rows are independent in the step kernel and in the prefill, so a row whose K / V caches were copied from another row
must continue exactly as that row's history run from scratch: the checks here are bitwise.
  1. fork equals re-run: an engine that selects rows mid-window gives, from then on, the logits of an engine that ran
     the reordered histories from the start - on the tiny golden priors, on a wide stack with every attn_func (6 and 7
     included) at 8 and 32 rows, and through the fp32 window;
  2. one prime: sampling n continuations of one given row equals sampling n copies of it;
  3. keep-best end to end: the log-probabilities a selecting window returns are those of its returned codes re-scored
     with their own conditioning (token_stats), within the prefill-against-stepping tolerance, in one window and over
     two windows of sample_level."""
import pytest
import torch

from golden_util import Fixture, rel_err

pytestmark = pytest.mark.gpu

TOL_PREFILL = 3e-3       # relative, prefill against stepping (tests/test_gpu_token_stats.py, DESIGN.md 5.2)


def _make_prior(fx):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae, make_prior
    c = fx.cfg
    vq = make_vqvae(setup_hparams(c["vq_name"], dict(restore_vqvae="", **c["vq_over"])), "cpu")
    prior = make_prior(setup_hparams(c["pr_name"], dict(restore_prior="", **c["pr_over"])), vq, "cpu")
    prior.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
    return prior.cuda().eval()


def _parents(N):
    """identity (row 0), a swap (1, 2), a 3-cycle (3, 4, 5), a broadcast of row 0 (6, 7); at 32 rows also a reversal
    of rows 8..29 and two more copies of row 9"""
    p = [0, 2, 1, 4, 5, 3, 0, 0]
    if N > 8:
        p += list(range(29, 7, -1)) + [9, 9]
    return p[:N]


def _rows(v, idx):
    return None if v is None else v[idx].contiguous()


def _engine_run(m, N, toks, x_cond, y_cond, enc, t0, t1, t2, parents=None, cont=None):
    """teacher-forced run on the fp16 engine: positions [0, t0) prefilled (stepped when the engine has no prefill),
    [t0, t1) stepped, then (parents) select and switch to the continuation tokens `cont`, then [t1, t2) stepped.
    Returns the logits of [t1, t2), fp32 [N, t2 - t1, bins]."""
    from jukebox_b200.transformer import f32
    eng = m._fresh_engine(N, enc)
    logits = torch.empty(N, t2 - t1, m.bins, device="cuda")
    buf = torch.empty(N, m.bins, device="cuda")

    def bias(xc):
        if not (m.add_cond_after_transformer and xc is not None and eng.has_logits_gemm):
            return None
        return f32.linear_nk(xc.reshape(-1, m.width), m.x_out.weight).view(N, xc.shape[1], m.bins)
    lb = bias(x_cond)
    if 1 < t0 <= eng.prefill_capacity:
        eng.prefill(N, t0, tokens=toks, y_cond=y_cond, x_cond=x_cond)
    else:
        for _ in range(t0):
            eng.step(N, tokens=toks, y_cond=y_cond, x_cond=x_cond)
    for t in range(t0, t2):
        if t == t1 and parents is not None:
            eng.select(parents)
            toks, x_cond, y_cond = cont, _rows(x_cond, parents), _rows(y_cond, parents)
            lb = bias(x_cond)
        eng.step(N, tokens=toks, y_cond=y_cond, x_cond=x_cond, logits=buf, logit_bias=lb)
        if t >= t1:
            logits[:, t - t1] = buf
    m.transformer.del_cache()
    return logits


def _fork_equals_rerun(m, N, toks, x_cond, y_cond, enc, t0, t1, t2, seed):
    parents = _parents(N)
    g = torch.Generator().manual_seed(seed)
    cont = toks[parents].clone()
    cont[:, t1:] = torch.randint(0, m.bins, (N, cont.shape[1] - t1), generator=g).cuda()
    forked = _engine_run(m, N, toks, x_cond, y_cond, enc, t0, t1, t2, parents, cont)
    rerun = _engine_run(m, N, cont, _rows(x_cond, parents), _rows(y_cond, parents), _rows(enc, parents), t0, t1, t2)
    assert bool(torch.isfinite(forked).all())
    assert torch.equal(forked, rerun), float((forked - rerun).abs().max())
    # and a selection really moved state: an engine that did not select continues differently
    plain = _engine_run(m, N, cont, x_cond, y_cond, enc, t0, t1, t2)
    assert not torch.equal(plain, rerun)


def _window_conds(prior, fx, N, seed):
    """N rows of tokens of a whole window (random ids) with the fixture's conditioning repeated row by row"""
    y = torch.from_numpy(fx["y"]).cuda() if "y" in fx else None
    z_conds = [torch.from_numpy(fx["z_cond"]).cuda()] if "z_cond" in fx else []
    tokens = torch.from_numpy(fx["tokens"]).cuda()
    z = prior.prior_postprocess(tokens) if prior.single_enc_dec else tokens
    rows = torch.arange(N, device="cuda") % z.shape[0]
    seq, x_cond, y_cond, enc, _, _ = prior._condition(z[rows], [c[rows] for c in z_conds],
                                                      None if y is None else y[rows], True)
    g = torch.Generator().manual_seed(seed)
    seq = torch.randint(0, prior.prior.bins, seq.shape, generator=g).cuda()
    return seq, x_cond, y_cond, enc


@pytest.mark.parametrize("N", [8, 32])
@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_fork_equals_rerun_on_the_golden_priors(tag, N):
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    seq, x_cond, y_cond, enc = _window_conds(prior, fx, N, seed=N)
    D = seq.shape[1]
    _fork_equals_rerun(prior.prior, N, seq, x_cond, y_cond, enc, D // 4, D // 2, D - 2, seed=N + 1)


def _wide_stack():
    """a stack with every attn_func: attn_order 11 (block, transpose, previous block; layer 15 encoder-decoder) with
    layer 4 made a prime layer"""
    from oracle.synth import synth_state_dict
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    m = ConditionalAutoregressive2D((384,), 320, width=1024, depth=16, heads=8, attn_order=11, blocks=16,
                                    x_cond=True, y_cond=True, encoder_dims=48, prime_len=40)
    blk = m.transformer._attn_mods[4]
    assert blk.attn_func == 2 and m.transformer._attn_mods[15].attn_func == 6
    blk.attn_func = blk.attn.attn_func = 7
    m.transformer._attn_mods[9].attn_func = m.transformer._attn_mods[9].attn.attn_func = 0
    named = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth_state_dict(named, 5).items()})
    m = m.cuda().eval()
    assert sorted({b.attn_func for b in m.transformer._attn_mods}) == [0, 1, 2, 3, 6, 7]
    return m


@pytest.mark.parametrize("N", [8, 32])
def test_fork_equals_rerun_with_every_attn_func(N):
    m = _wide_stack()
    g = torch.Generator().manual_seed(7)
    toks = torch.randint(0, m.bins, (N, m.input_dims), generator=g).cuda()
    x_cond = (torch.randn(N, m.input_dims, m.width, generator=g) * 0.3).cuda()
    y_cond = (torch.randn(N, 1, m.width, generator=g) * 0.3).cuda().view(N, m.width)
    enc = (torch.randn(N, 48, m.width, generator=g) * 0.5).cuda()
    # blocks of 24 positions: t1 inside a block, t2 two blocks on (block, previous-block and prime layers all move)
    _fork_equals_rerun(m, N, toks, x_cond, y_cond, enc, 30, 61, 110, seed=N)


@pytest.mark.parametrize("tag", ["single_enc_dec", "upsampler"])
def test_fork_equals_rerun_in_the_fp32_window(tag):
    from jukebox_b200.prior.autoregressive import SamplingWindowF32
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    m = prior.prior
    N = 8
    seq, x_cond, y_cond, enc = _window_conds(prior, fx, N, seed=3)
    D = seq.shape[1]
    t1, t2 = D // 2, D - 2
    parents = _parents(N)
    yc = None if y_cond is None else y_cond.view(N, 1, -1)

    def window(toks, xc, ycc, e):
        return SamplingWindowF32(m, N, toks[:, :t2], xc, ycc, e, False, 1.0, 0, 0.0, True, t2 + 1)
    w = window(seq, x_cond, yc, enc)
    w.advance(t1)
    w.select(parents)
    g = torch.Generator().manual_seed(4)
    cont = w.tokens.clone()
    cont[:, t1:t2] = torch.randint(0, m.bins, (N, t2 - t1), generator=g).cuda()
    w.tokens[:, t1:t2] = cont[:, t1:t2]
    assert w.ancestry.tolist() == parents
    w.advance(t2)
    forked = w.preds[:, t1:t2].clone()
    m.transformer.del_cache()
    r = window(cont, _rows(x_cond, parents), _rows(yc, parents), _rows(enc, parents))
    r.advance(t2)
    rerun = r.preds[:, t1:t2].clone()
    m.transformer.del_cache()
    assert torch.equal(forked, rerun), float((forked - rerun).abs().max())
    assert torch.equal(w.tokens[:, :t1], seq[parents, :t1])


@pytest.mark.parametrize("fp16", [True, False])
@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_one_prime_equals_its_copies(tag, fp16):
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    N = 5
    y = torch.from_numpy(fx["y"]).cuda()[:1] if "y" in fx else None
    z_conds = [torch.from_numpy(fx["z_cond"]).cuda()[:1]] if "z_cond" in fx else []
    tokens = torch.from_numpy(fx["tokens"]).cuda()
    z = (prior.prior_postprocess(tokens) if prior.single_enc_dec else tokens)[:1, :prior.n_ctx // 3].contiguous()
    rep = lambda v: None if v is None else v.repeat(N, *[1] * (v.dim() - 1))
    torch.manual_seed(9)
    one = prior.sample(N, z=z, z_conds=z_conds, y=y, fp16=fp16, temp=0.9, get_logprobs=True)
    torch.manual_seed(9)
    many = prior.sample(N, z=rep(z), z_conds=[rep(c) for c in z_conds], y=rep(y), fp16=fp16, temp=0.9,
                        get_logprobs=True)
    assert torch.equal(one[0], many[0]) and torch.equal(one[1], many[1])
    assert torch.equal(one[0][:, :z.shape[1]], rep(z))
    assert len({tuple(r) for r in one[0].tolist()}) > 1, "the continuations differ per row"
    # keep-best on top of one prime: every row descends from the one given item
    torch.manual_seed(9)
    codes, anc = prior.sample(N, z=z, z_conds=z_conds, y=y, fp16=fp16, temp=0.9, select_every=4, select_keep=2)
    assert anc.tolist() == [0] * N and codes.shape == one[0].shape


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_keep_best_window_matches_its_rescored_codes(tag):
    """A log-probability is z - lse, so it moves by at most twice a logit's error: the bound is 2 TOL_PREFILL max|z|
    (max|z| from the fp32 path), as tests/test_gpu_token_stats.py bounds token_stats against the oracle.
    A single_enc_dec prior is checked on its token sequence (ConditionalAutoregressive2D.primed_sample / token_stats):
    its sampler may draw an id of the lyric vocabulary, which SimplePrior returns as code 0, and re-scoring code 0
    would condition every later position on another history."""
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    m = prior.prior
    N = 6
    g = torch.Generator().manual_seed(2)
    y0 = torch.from_numpy(fx["y"]).cuda() if "y" in fx else None
    zc0 = [torch.from_numpy(fx["z_cond"]).cuda()] if "z_cond" in fx else []
    rows = torch.arange(N, device="cuda") % (y0.shape[0] if y0 is not None else zc0[0].shape[0] if zc0 else 1)
    y = None if y0 is None else y0[rows]
    z_conds = [c[rows] for c in zc0]
    if z_conds:       # upper-level codes differ per row, so a row continued from another row's state would show
        z_conds = [torch.randint(0, prior.l_bins, c.shape, generator=g).cuda() for c in z_conds]
    P = prior.n_ctx // 4
    z = torch.randint(0, prior.l_bins, (N, P), generator=g).cuda()
    sel = dict(fp16=True, temp=1.0, get_logprobs=True, select_every=5, select_keep=2)
    torch.manual_seed(5)
    if prior.single_enc_dec:
        seq, x_cond, y_cond, _, _, _ = prior._condition(z, z_conds, y, True)
        out, lp, anc = m.primed_sample(N, seq, x_cond, y_cond, **sel)
        assert torch.equal(out[:, :seq.shape[1]], seq[anc])

        def rescore(idx):
            return m.token_stats(out, x_cond[idx], y_cond[idx]).logp

        with torch.no_grad():
            scale = float(m(out, x_cond[anc], y_cond[anc], fp16=False, get_preds=True)[1].abs().max())
    else:
        codes, lp, anc = prior.sample(N, z=z, z_conds=z_conds, y=y, **sel)
        assert torch.equal(codes[:, :P], z[anc])

        def rescore(idx):
            return prior.token_stats(codes, [c[idx] for c in z_conds], None if y is None else y[idx]).logp

        with torch.no_grad():
            seq, x_cond, y_cond, enc, _, _ = prior._condition(codes, [c[anc] for c in z_conds],
                                                              None if y is None else y[anc], False)
            scale = float(m(seq, x_cond, y_cond, enc, fp16=False, get_preds=True)[1].abs().max())
    assert sorted(set(anc.tolist())) != list(range(N)), "selection copied rows"
    bound = 2 * TOL_PREFILL * scale
    d = float((lp - rescore(anc)).abs().max())
    print(f"prior_{tag}: keep-best window against its re-scored tokens: |dlogp| {d:.2e} (bound {bound:.2e}), "
          f"ancestry {anc.tolist()}")
    assert d <= bound
    # a wrong history is far off: the same codes scored as if every row descended from its own input item
    if z_conds:
        assert float((lp - rescore(torch.arange(N, device="cuda"))).abs().max()) > 3 * bound


def test_keep_best_over_two_windows_of_sample_level():
    from jukebox_b200.sample import plan_windows, sample_level, song_token_stats
    fx = Fixture("prior_upsampler")
    prior = _make_prior(fx)
    n, n_ctx = 4, prior.n_ctx
    hop = n_ctx // 2
    T = n_ctx + hop
    assert len(plan_windows(0, T, n_ctx, hop)) == 2
    g = torch.Generator().manual_seed(12)
    zs = [torch.zeros(n, 0, dtype=torch.long, device="cuda"),
          torch.randint(0, prior.l_bins, (n, T // prior.cond_downsample), generator=g).cuda()]
    upper0 = zs[1].clone()
    labels = dict(y=torch.zeros(n, 0, dtype=torch.long), info=[{}] * n)
    lp_song = torch.full((n, T), float("nan"), device="cuda")
    sample = prior.sample
    seen, state = [], dict(i0=0)

    def recording_sample(**kw):              # the sampler's own log-probabilities, rows following the ancestry
        codes, lp, anc = sample(get_logprobs=True, **kw)
        i0, k = state["i0"], len(anc)
        have, new = zs[0].shape[1], codes.shape[1] - kw["z"].shape[1]
        lp_song[i0:i0 + k] = lp_song[i0:i0 + k][anc]
        lp_song[i0:i0 + k, have:have + new] = lp[:, -new:]
        state["i0"] = (i0 + k) % n
        seen.append(anc.tolist())
        return codes, anc
    prior.sample = recording_sample
    try:
        torch.manual_seed(6)
        sample_level(zs, labels, dict(max_batch_size=2, fp16=True, temp=1.0, select_every=6, select_keep=1), 0, prior,
                     T, hop, None)
    finally:
        del prior.sample
    assert zs[0].shape == (n, T) and bool(torch.isfinite(lp_song).all())
    assert len(seen) == 4 and any(a != [0, 1] for a in seen)
    # the upper level followed its items: each piece's rows are rows of its own input
    for i0 in (0, 2):
        own = set(map(tuple, upper0[i0:i0 + 2].tolist()))
        assert all(tuple(r) in own for r in zs[1][i0:i0 + 2].tolist())
    assert not torch.equal(zs[1], upper0)
    st = song_token_stats(prior, zs, labels, 0, hop, max_batch_size=4)
    e = rel_err(st.logp.cpu().numpy(), lp_song.cpu().numpy())
    print(f"keep-best over two windows of sample_level: rel {e:.2e}, ancestries {seen}")
    assert e < TOL_PREFILL


def test_select_rejects_bad_calls():
    from oracle.synth import synth_state_dict
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    m = ConditionalAutoregressive2D((64,), 32, width=256, depth=3, heads=2, attn_order=2, blocks=8)
    named = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth_state_dict(named, 3).items()})
    m = m.cuda().eval()
    eng = m._fresh_engine(4, None)
    assert eng.prefill_capacity >= 8
    with pytest.raises(RuntimeError, match="outside"):
        eng.select([0, 1, 2, 4])
    with pytest.raises(RuntimeError, match="out of range"):
        eng.select([0] * 5)
    info = eng.select([1, 0, 2, 3])             # a swap allocates its workspace
    assert info.n_stash == 2 and info.workspace_bytes == 2 * info.row_bytes
    toks = torch.zeros(4, m.input_dims, dtype=torch.long, device="cuda")
    xc = torch.zeros(4, m.input_dims, m.width, device="cuda") if m.x_cond else None
    yc = torch.zeros(4, m.width, device="cuda") if m.y_cond else None
    eng.prefill(4, 8, tokens=toks, x_cond=xc, y_cond=yc, n_layers=1)
    with pytest.raises(RuntimeError, match="stopped early"):
        eng.select([0, 0, 0, 0])
    m.transformer.del_cache()
    eng.select([0, 0, 0, 0])                    # after a reset the rows are whole again
