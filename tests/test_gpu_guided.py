"""Guided sampling on the GPU (jk_sample_guided, csrc/sampling.cu; guided windows, prior/autoregressive.py).

  1. the fused launch against its composition - torch g = c + s * (c - u), then jk_filter_logits, then
     jk_sample_categorical(_scored) - bit for bit in both token rows and in logp, over s, temp, the filters, ragged
     and power-of-two bins up to 4096, 1 and 16 pairs and strided rows; untouched cells stay untouched; s = 0 is the
     unguided draw of c; and the draws follow softmax(g / T);
  2. a guided window at scale 1 is, bit for bit, the first N rows of an unguided window of 2N rows whose last N rows
     carry the alternative conditioning (the golden tiny priors and a stack with every attn_func, fp16 and fp32);
  3. at another scale each drawn token is the composed draw from the window's own c and u rows, and the u rows are the
     logits of a teacher-forced pass under the alternative conditioning;
  4. keep-best selection moves pairs together and its log-likelihoods re-score; sample_level carries guidance labels."""
import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err

pytestmark = pytest.mark.gpu

TOL_PREFILL = 3e-3       # relative, prefill against stepping (tests/test_gpu_token_stats.py, DESIGN.md 5.2)


def _composed(c, u, s, temp, top_k, top_p, seed, pos, tokens, logp):
    from jukebox_b200.transformer.ops import filter_logits_scaled, sample_categorical_scored
    g = c + s * (c - u)
    if top_k or top_p:
        sample_categorical_scored(filter_logits_scaled(g, temp, top_k, top_p), c, 1.0, seed, pos, tokens, logp)
    else:
        sample_categorical_scored(g, c, temp, seed, pos, tokens, logp)


def test_fused_launch_equals_its_composition():
    from jukebox_b200.transformer.ops import sample_guided
    gen = torch.Generator(device="cuda").manual_seed(1)
    L, checked = 9, 0
    for bins in (80, 2048, 2127, 4096):
        for n in (1, 16):
            # strided operands: c and u are column windows of wider buffers, token rows of a taller poisoned tensor
            cbuf = torch.randn(n, bins + 40, device="cuda", generator=gen) * 3
            ubuf = torch.randn(n, bins + 17, device="cuda", generator=gen) * 3
            c, u = cbuf[:, 5:5 + bins], ubuf[:, 1:1 + bins]
            for s in (0.0, -0.5, 2.0):
                for temp in (0.7, 1.0):
                    for top_k, top_p in ((0, 0.0), (min(40, bins), 0.0), (0, 0.9)):
                        pos, seed = (checked * 7) % L, 1000 + checked
                        toks = torch.full((2 * n + 3, L), -7, dtype=torch.long, device="cuda")
                        logp = torch.full((n + 2, L + 3), -9.0, device="cuda")
                        before_t, before_l = toks.clone(), logp.clone()
                        a, b = toks[1:n + 1], toks[n + 2:2 * n + 2]
                        sample_guided(c, u, s, temp, top_k, top_p, seed, pos, a, b, logp[1:n + 1, 2:2 + L])
                        ref_t = torch.zeros(n, L, dtype=torch.long, device="cuda")
                        ref_l = torch.zeros(n, L, device="cuda")
                        _composed(c, u, s, temp, top_k, top_p, seed, pos, ref_t, ref_l)
                        case = (bins, n, s, temp, top_k, top_p)
                        assert torch.equal(a[:, pos], ref_t[:, pos]), case
                        assert torch.equal(b[:, pos], ref_t[:, pos]), case
                        assert torch.equal(logp[1:n + 1, 2 + pos], ref_l[:, pos]), case
                        # every other cell and row is untouched
                        mask = torch.ones_like(toks, dtype=torch.bool)
                        mask[1:n + 1, pos] = mask[n + 2:2 * n + 2, pos] = False
                        assert torch.equal(toks[mask], before_t[mask]), case
                        lmask = torch.ones_like(logp, dtype=torch.bool)
                        lmask[1:n + 1, 2 + pos] = False
                        assert torch.equal(logp[lmask], before_l[lmask]), case
                        checked += 1
    assert checked == 4 * 2 * 3 * 2 * 3


def test_weight_zero_is_the_unguided_draw():
    from jukebox_b200.transformer.ops import filter_logits_scaled, sample_categorical, sample_guided
    gen = torch.Generator(device="cuda").manual_seed(2)
    for bins in (80, 2127):
        c = torch.randn(16, bins, device="cuda", generator=gen) * 2
        u = torch.randn(16, bins, device="cuda", generator=gen) * 2
        for top_k, temp in ((0, 0.9), (30, 1.0)):
            a = torch.zeros(16, 64, dtype=torch.long, device="cuda")
            b, ref = torch.zeros_like(a), torch.zeros_like(a)
            for pos in range(64):
                sample_guided(c, u, 0.0, temp, top_k, 0.0, 77, pos, a, b)
                if top_k:
                    sample_categorical(filter_logits_scaled(c, temp, top_k, 0.0), 1.0, 77, pos, ref)
                else:
                    sample_categorical(c, temp, 77, pos, ref)
            assert torch.equal(a, ref) and torch.equal(b, ref)
            assert len(set(a.view(-1).tolist())) > 4


def test_guided_draws_follow_softmax_of_g():
    from scipy.stats import chi2
    from jukebox_b200.transformer.ops import sample_guided
    n, bins, temp, s = 16, 64, 0.8, 1.5
    gen = torch.Generator(device="cuda").manual_seed(3)
    crow = torch.randn(bins, device="cuda", generator=gen)
    urow = torch.randn(bins, device="cuda", generator=gen)
    c, u = crow.expand(n, bins).contiguous(), urow.expand(n, bins).contiguous()
    P = 4096
    a = torch.zeros(n, P, dtype=torch.long, device="cuda")
    b = torch.zeros_like(a)
    for pos in range(P):
        sample_guided(c, u, s, temp, 0, 0.0, 123, pos, a, b)
    assert torch.equal(a, b)
    toks = a.cpu().numpy().reshape(-1)
    counts = np.bincount(toks, minlength=bins).astype(np.float64)
    g = crow.double().cpu() + s * (crow.double().cpu() - urow.double().cpu())
    p = torch.softmax(g / temp, 0).numpy()
    expect = counts.sum() * p
    keep = expect >= 5          # the rare bins pooled into one cell
    obs = np.append(counts[keep], counts[~keep].sum())
    exp = np.append(expect[keep], expect[~keep].sum())
    stat = float(((obs - exp) ** 2 / np.maximum(exp, 1e-9)).sum())
    dof = len(obs) - 1
    pval = float(chi2.sf(stat, dof))
    print(f"guided draws: chi2 {stat:.1f} on {dof} dof, p {pval:.3f}")
    assert pval > 1e-4
    # and not the distribution of c alone
    pc = torch.softmax(crow.double().cpu() / temp, 0).numpy()
    assert float(((counts - counts.sum() * pc) ** 2 / (counts.sum() * pc)).sum()) > 10 * dof


# ---- windows ------------------------------------------------------------------------------------------------------
def _make_prior(fx, **over):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae, make_prior
    c = fx.cfg
    vq = make_vqvae(setup_hparams(c["vq_name"], dict(restore_vqvae="", **c["vq_over"])), "cpu")
    prior = make_prior(setup_hparams(c["pr_name"], dict(restore_prior="", **c["pr_over"], **over)), vq, "cpu")
    prior.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
    return prior.cuda().eval()


def _golden_case(tag, N, seed):
    """(model, given tokens [N, P], their alternative [N, P], conds, alternative conds, sample_tokens): the fixture's
    conditioning on the rows, the alternative from other label / upper-code rows"""
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    g = torch.Generator().manual_seed(seed)
    rows = torch.arange(N) % 2
    y = torch.from_numpy(fx["y"])[rows].cuda() if "y" in fx else None
    zc = [torch.randint(0, prior.l_bins, (N, prior.n_ctx // prior.cond_downsample), generator=g).cuda()] \
        if "z_cond" in fx else []
    z = torch.randint(0, prior.l_bins, (N, prior.n_ctx), generator=g).cuda()
    seq, xc, yc, enc, _, pl = prior._condition(z, zc, y, True)
    if y is not None:     # other artists / genres and lyrics
        y_alt = y.clone()
        y_alt[:, 3] = (y[:, 3] + 1) % 10
        y_alt[:, 4] = (y[:, 4] + 3) % 10
        if prior.n_tokens:
            y_alt[:, -prior.n_tokens:] = torch.randint(1, 40, (N, prior.n_tokens), generator=g).cuda()
        seq_a, xa, ya, ea, _, _ = prior._condition(z, zc, y_alt, True)
    else:                 # the upsampler has no labels: other upper-level codes
        zc_a = [torch.randint(0, prior.l_bins, c.shape, generator=g).cuda() for c in zc]
        seq_a, xa, ya, ea, _, _ = prior._condition(z, zc_a, y, True)
    P = pl + prior.n_ctx // 4
    return prior.prior, seq[:, :P], seq_a[:, :P], (xc, yc, enc), (xa, ya, ea), seq.shape[1]


def _wide_case(N, seed):
    from oracle.synth import synth_state_dict
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    m = ConditionalAutoregressive2D((384,), 320, width=1024, depth=16, heads=8, attn_order=11, blocks=16,
                                    x_cond=True, y_cond=True, encoder_dims=48, prime_len=40)
    blk = m.transformer._attn_mods[4]
    blk.attn_func = blk.attn.attn_func = 7
    m.transformer._attn_mods[9].attn_func = m.transformer._attn_mods[9].attn.attn_func = 0
    named = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth_state_dict(named, 5).items()})
    m = m.cuda().eval()
    assert sorted({b.attn_func for b in m.transformer._attn_mods}) == [0, 1, 2, 3, 6, 7]
    g = torch.Generator().manual_seed(seed)

    def conds():
        return ((torch.randn(N, m.input_dims, m.width, generator=g) * 0.3).cuda(),
                (torch.randn(N, 1, m.width, generator=g) * 0.3).cuda(),
                (torch.randn(N, 48, m.width, generator=g) * 0.5).cuda())
    prime = torch.randint(0, m.bins, (N, 50), generator=g).cuda()
    return m, prime, prime, conds(), conds(), 120


def _case(tag, N, seed):
    return _wide_case(N, seed) if tag == "every_attn_func" else _golden_case(tag, N, seed)


def _cat(a, b):
    return None if a is None else torch.cat([a, b])


@pytest.mark.parametrize("fp16", [True, False])
@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler", "every_attn_func"])
def test_scale_one_is_the_unguided_window_of_2n_rows(tag, fp16):
    N = 3
    m, x, x_alt, (xc, yc, enc), (xa, ya, ea), T = _case(tag, N, seed=11)
    how = dict(fp16=fp16, temp=0.9, sample_tokens=T, get_logprobs=True)
    torch.manual_seed(4)
    z, lp = m.primed_sample(N, x, xc, yc, enc, guidance_scale=1.0, x_cond_alt=xa, y_cond_alt=ya, encoder_kv_alt=ea,
                            x_alt=x_alt, **how)
    torch.manual_seed(4)
    z2, lp2 = m.primed_sample(2 * N, torch.cat([x, x_alt]), _cat(xc, xa), _cat(yc, ya), _cat(enc, ea), **how)
    assert torch.equal(z, z2[:N]) and torch.equal(lp, lp2[:N])
    assert torch.equal(z[:, :x.shape[1]], x) and z.shape == (N, T)
    assert len({tuple(r) for r in z[:, x.shape[1]:].tolist()}) > 1


@pytest.mark.parametrize("fp16", [True, False])
@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_drawn_tokens_are_the_composed_draw_of_the_windows_rows(tag, fp16):
    from jukebox_b200.prior.autoregressive import Guide, SamplingWindow, SamplingWindowF32
    from jukebox_b200.transformer.ops import filter_logits_scaled, sample_categorical
    N, scale, temp, top_p = 4, 3.0, 0.95, 0.9
    m, x, x_alt, (xc, yc, enc), (xa, ya, ea), T = _golden_case(tag, N, seed=5)
    P = x.shape[1]
    cls = SamplingWindow if fp16 else SamplingWindowF32
    torch.manual_seed(8)
    win = cls(m, N, x, xc, yc, enc, fp16, temp, 0, top_p, True, T, guide=Guide(scale, xa, ya, ea, x_alt))
    win.advance(T)
    z, preds = win.finish()
    assert torch.equal(preds, win.preds[:N]) and torch.equal(z, win.tokens[:N])
    ref = torch.zeros(N, T, dtype=torch.long, device="cuda")
    for t in range(P, T):
        c, u = win.preds[:N, t], win.preds[N:, t]
        sample_categorical(filter_logits_scaled(c + (scale - 1) * (c - u), temp, 0, top_p), 1.0, win.seed, t, ref)
    assert torch.equal(win.tokens[:N, P:], ref[:, P:])
    assert torch.equal(win.tokens[N:, P:], ref[:, P:]) and torch.equal(win.tokens[N:, :P], x_alt)
    # the u rows are the alternative conditioning's logits at the returned codes (a teacher-forced pass)
    alt_seq = torch.cat([x_alt, z[:, P:]], 1)
    _, want = m(alt_seq, xa, ya, ea, fp16=fp16, get_preds=True)
    e = rel_err(win.preds[N:].cpu().numpy(), want.cpu().numpy())
    _, want_c = m(z, xc, yc, enc, fp16=fp16, get_preds=True)
    ec = rel_err(win.preds[:N].cpu().numpy(), want_c.cpu().numpy())
    print(f"{tag} fp16={fp16}: u rows against a teacher-forced pass {e:.2e}, c rows {ec:.2e}")
    assert e < TOL_PREFILL and ec < TOL_PREFILL
    # guidance moved the draws: the unguided window of the same seed draws other tokens
    torch.manual_seed(8)
    plain = m.primed_sample(N, x, xc, yc, enc, fp16=fp16, temp=temp, top_p=top_p, sample_tokens=T)
    assert not torch.equal(plain, z)


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_keep_best_moves_pairs_and_rescores(tag):
    from jukebox_b200.prior.autoregressive import Guide, SamplingWindow
    N = 6
    m, x, x_alt, (xc, yc, enc), (xa, ya, ea), T = _golden_case(tag, N, seed=9)
    P = x.shape[1]
    torch.manual_seed(3)
    win = SamplingWindow(m, N, x, xc, yc, enc, True, 1.0, 0, 0.0, False, T, get_logprobs=True, select_every=5,
                         select_keep=2, guide=Guide(2.0, xa, ya, ea, x_alt))
    win.advance(T)
    z, lp, anc = win.finish()
    assert sorted(set(anc.tolist())) != list(range(N)), "selection copied rows"
    # each alternative row is its item's: its given tokens and conditioning, the pair's drawn tokens
    assert torch.equal(win.tokens[N:, :P], x_alt[anc]) and torch.equal(win.tokens[N:, P:], z[:, P:])
    assert torch.equal(z[:, :P], x[anc]) and torch.equal(win.ancestry[N:], anc)
    for mine, a, b in ((win.x_cond, xc, xa), (win.y_cond, yc, ya)):
        if a is not None:
            assert torch.equal(mine[:N].view(a[anc].shape), a[anc].float())
            assert torch.equal(mine[N:].view(b[anc].shape), b[anc].float())
    st = m.token_stats(z, xc[anc], None if yc is None else yc[anc], None if enc is None else enc[anc])
    with torch.no_grad():
        scale = float(m(z, xc[anc], None if yc is None else yc[anc], None if enc is None else enc[anc], fp16=False,
                        get_preds=True)[1].abs().max())
    d = float((lp - st.logp).abs().max())
    print(f"{tag}: guided keep-best against its re-scored tokens |dlogp| {d:.2e} (bound {2 * TOL_PREFILL * scale:.2e})")
    assert d <= 2 * TOL_PREFILL * scale


def test_sample_level_with_guidance_labels():
    from jukebox_b200.sample import plan_windows, sample_level, null_labels
    fx = Fixture("prior_upsampler")
    labelled = dict(labels=True, labels_v3=True, y_bins=(10, 100), max_bow_genre_size=1, t_bins=64)
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae, make_prior
    from oracle.synth import synth_state_dict
    c = fx.cfg
    vq = make_vqvae(setup_hparams(c["vq_name"], dict(restore_vqvae="", **c["vq_over"])), "cpu")
    prior = make_prior(setup_hparams(c["pr_name"], dict(c["pr_over"], restore_prior="", **labelled)), vq, "cpu")
    named = [(k, tuple(v.shape)) for k, v in prior.state_dict().items()]
    prior.load_state_dict({k: torch.from_numpy(v) for k, v in synth_state_dict(named, 6).items()})
    prior = prior.cuda().eval()
    n, n_ctx = 3, prior.n_ctx
    hop = n_ctx // 2
    T = 2 * n_ctx
    assert len(plan_windows(0, T, n_ctx, hop)) == 3
    g = torch.Generator().manual_seed(13)
    zs = [torch.zeros(n, 0, dtype=torch.long, device="cuda"),
          torch.randint(0, prior.l_bins, (n, T // prior.cond_downsample), generator=g).cuda()]
    total = T * prior.raw_to_tokens
    meta = lambda a, gg: dict(artist=a, genre=gg, lyrics="", total_length=total, offset=0)
    labels = prior.labeller.get_batch_labels([meta("a", "b")] * n, "cuda")
    labels["y"][:, 3], labels["y"][:, 4] = torch.tensor([3, 4, 5]), torch.tensor([7, 8, 9])
    guide = prior.labeller.get_batch_labels([meta("c", "d")] * n, "cuda")
    guide["y"][:, 3], guide["y"][:, 4] = 6, 1
    sample, seen = prior.sample, []

    def recording(**kw):
        seen.append((torch.get_rng_state(), kw))
        return sample(**kw)
    prior.sample = recording
    try:
        torch.manual_seed(6)
        sample_level(zs, labels, dict(max_batch_size=2, fp16=True, temp=1.0, guidance_scale=2.0, guidance_labels=guide),
                     0, prior, T, hop, None)
        z_guided = zs[0].clone()
        zs[0] = zs[0][:, :0]
        torch.manual_seed(6)
        sample_level(zs, labels, dict(max_batch_size=2, fp16=True, temp=1.0, guidance_scale=2.0), 0, prior, T, hop,
                     None)
    finally:
        del prior.sample
    assert z_guided.shape == (n, T) and zs[0].shape == (n, T)
    assert len(seen) == 12 and all(kw["guidance_scale"] == 2.0 for _, kw in seen)
    starts = [w.start for w in plan_windows(0, T, n_ctx, hop)]
    for i, (state, kw) in enumerate(seen):
        w, piece = (i % 6) // 2, i % 2
        src = guide if i < 6 else null_labels(prior, labels)
        want = prior.get_y(src, starts[w])[2 * piece:2 * piece + 2]
        assert torch.equal(kw["guidance_y"], want), i
        assert torch.equal(kw["y"], prior.get_y(labels, starts[w])[2 * piece:2 * piece + 2]), i
    # a replayed window call draws the same codes: the level hands the prior exactly these arguments
    state, kw = seen[2]
    torch.set_rng_state(state)
    again = prior.sample(**kw)
    w1 = starts[1]
    assert torch.equal(again[:, n_ctx - hop:], z_guided[:2, w1 + n_ctx - hop:w1 + n_ctx])
    assert not torch.equal(z_guided, zs[0]), "the null labels and the guidance labels guide differently"
