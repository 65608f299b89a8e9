"""Token statistics on the GPU: jk_xout_stats (fused x_out + entropy + top-k, csrc/score.cu) against the fp64 oracle at
the tile edges, exact ties, batch independence and bit-identity with jk_xout_logprob; SimplePrior.token_stats against
the oracle transformer's logits; song_token_stats against the log-probabilities the sampler returned while drawing the
same codes, window by window.

Tolerances.  TOL_LOGP (tests/test_gpu_score.py, derived in DESIGN.md 5.2) bounds |logp - fp64| for logits within
|z| <~ 30; logp = z - lse, so it covers twice the error eps of a logit.  To first order the entropy moves by
dH = -sum_b p_b (log p_b + H) dz_b, so |dH| <= eps E_p|S - H| with S = -log p the surprisal.  E_p|S - H| is at most
the standard deviation of S, and the variance of the surprisal over n outcomes is below ln^2(n - 1) / 4 + 1 (15.7 at
n = 2127), so |dH| < 4 eps <= 2 TOL_LOGP; the fp64 combine adds rounding far below that (TOL_H_ROUND covers the fp32
u sums and the final fp32 rounding of H).  A top-k id may differ from fp64 only where the fp64 logits of neighbouring
ranks are within 2 eps <= TOL_LOGP of each other: the check is that the fp64 logit of the id returned at rank j lies
within TOL_LOGP of the fp64 rank-j logit, and that the returned ids are distinct."""
import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err
from oracle import score_np, stats_np

pytestmark = pytest.mark.gpu

TOL_LOGP = 2e-5          # nats: tests/test_gpu_score.py
TOL_H_ROUND = 1e-6       # nats: fp32 u partials and the fp32 result of the fp64 combine, for H up to ~8
TOL_H = 2 * TOL_LOGP + TOL_H_ROUND
TOL_PREFILL = 3e-3       # relative, prefill against stepping (tests/test_gpu_prefill.py TOL): the sampler steps


def _case(W, bins, M, seed):
    """activations with logits of std ~3 and every fifth row twice that (|z| up to ~30, as tests/test_gpu_score.py)"""
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(M, W, generator=g, dtype=torch.float64)
    h[::5] *= 2.0
    w = torch.randn(bins, W, generator=g, dtype=torch.float64) * (3.0 / W ** 0.5)
    tg = torch.randint(0, bins, (M,), generator=g)
    tg[0] = bins - 1
    return h.float(), w.float(), tg


def _check_topk(ids, tlp, z, lse, k, where):
    """ids / tlp [M, k] from the GPU against the fp64 logits z [M, bins] and lse [M]"""
    zs = -np.sort(-z, axis=-1)[:, :k]
    got_z = np.take_along_axis(z, ids, -1)
    assert (ids >= 0).all() and (ids < z.shape[1]).all(), where
    assert all(len(set(r)) == k for r in ids.tolist()), where
    d = float(np.abs(got_z - zs).max())
    assert d <= TOL_LOGP, (where, d)
    dl = float(np.abs(tlp - (got_z - lse[:, None])).max())
    assert dl <= TOL_LOGP, (where, dl)
    return d, dl


@pytest.mark.parametrize("W", [64, 1920, 4800])
def test_xout_stats_against_fp64(W):
    from jukebox_b200.score import xout_stats, xout_logprob
    worst = dict(logp=0.0, H=0.0, topz=0.0)
    for bins in (80, 128, 2048, 2127):
        for M in (1, 127, 128, 129, 300):
            h, w, tg = _case(W, bins, M, seed=W + bins + M)
            hg, wg, tgg = h.cuda(), w.cuda(), tg.cuda()
            for k in (1, 5, 16):
                lp, H, ids, tlp, lse, z = stats_np.xout_stats(h.double().numpy(), w.double().numpy(), tg.numpy(), k)
                st = xout_stats(hg, wg, tgg, top_k=k)
                dlp = float(np.abs(st.logp.cpu().double().numpy() - lp).max())
                dH = float(np.abs(st.entropy.cpu().double().numpy() - H).max())
                dlse = float(np.abs(st.lse.cpu().double().numpy() - lse).max())
                assert dlp <= TOL_LOGP and dlse <= TOL_LOGP and dH <= TOL_H, (W, bins, M, k, dlp, dlse, dH)
                dz, _ = _check_topk(st.topk_ids.cpu().numpy(), st.topk_logp.cpu().double().numpy(), z, lse, k,
                                    (W, bins, M, k))
                worst["logp"], worst["H"], worst["topz"] = max(worst["logp"], dlp), max(worst["H"], dH), max(worst["topz"], dz)
            # logp and lse are xout_logprob's bit for bit, with or without top-k; targets may be left out
            lp0, lse0 = xout_logprob(hg, wg, tgg, get_lse=True)
            assert torch.equal(st.logp, lp0) and torch.equal(st.lse, lse0), (W, bins, M)
            st0 = xout_stats(hg, wg)
            assert st0.logp is None and st0.topk_ids is None and st0.topk_logp is None
            assert torch.equal(st0.lse, lse0) and torch.equal(st0.entropy, st.entropy), (W, bins, M)
            if M == 300:
                for r in (0, 129, 299):          # a row alone gives the bits it gives in the batch
                    one = xout_stats(hg[r:r + 1], wg, tgg[r:r + 1], top_k=16)
                    for a, b in zip(one, st):
                        assert torch.equal(a, b[r:r + 1]), (W, bins, r)
    print(f"xout_stats W={W}: max |dlogp| {worst['logp']:.2e}, |dH| {worst['H']:.2e}, "
          f"top-k |dz| at rank {worst['topz']:.2e} (nats)")


@pytest.mark.parametrize("bins", [80, 2127])
def test_xout_stats_exact_ties_go_to_the_lower_id(bins):
    """duplicated x_out rows give bit-equal logits: within a bin tile, across bin tiles and in the ragged tail"""
    from jukebox_b200.score import xout_stats
    W, M = 256, 130
    h, w, _ = _case(W, bins, M, seed=bins)
    h[:, :] = h[:1]                              # every row the same: the same winners everywhere
    z = h[:1].double() @ w.double().T
    top = int(z.argmax())
    dups = [d for d in (3, 77, 129, 1000, bins - 1) if d < bins and d != top]
    for d in dups:
        w[d] = w[top]
    st = xout_stats(h.cuda(), w.cuda(), top_k=len(dups) + 2)
    ids = st.topk_ids.cpu()
    want = sorted([top] + dups)
    assert ids[:, :len(want)].tolist() == [want] * M, ids[0].tolist()
    assert (st.topk_logp[:, :len(want)] == st.topk_logp[:, :1]).all()
    zd = z[0].numpy().copy()
    zd[want] = -np.inf
    assert int(ids[0, len(want)]) == int(np.argmax(zd))


def test_xout_stats_rejects_what_the_split_cannot_hold():
    from jukebox_b200.score import xout_stats
    h, w, tg = _case(1024, 2127, 200, seed=1)
    hg, wg, tgg = h.cuda(), w.cuda(), tg.cuda()
    bad = hg.clone()
    bad[17, 3] = float("inf")
    with pytest.raises(RuntimeError, match="fp16 split"):
        xout_stats(bad, wg, tgg, top_k=4)
    tbad = tgg.clone()
    tbad[3] = -1
    with pytest.raises(RuntimeError, match="target"):
        xout_stats(hg, wg, tbad, top_k=4)
    st = xout_stats(hg, wg, tgg, top_k=4)
    assert bool(torch.isfinite(st.entropy).all()) and bool((st.topk_ids >= 0).all())


def _make_prior(fx):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae, make_prior
    c = fx.cfg
    vq = make_vqvae(setup_hparams(c["vq_name"], dict(restore_vqvae="", **c["vq_over"])), "cpu")
    prior = make_prior(setup_hparams(c["pr_name"], dict(restore_prior="", **c["pr_over"])), vq, "cpu")
    prior.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
    return prior.cuda().eval()


@pytest.mark.parametrize("D", [None, 40])
@pytest.mark.parametrize("tag", ["single_enc_dec", "upsampler"])
def test_prior_token_stats_against_the_oracle(tag, D):
    """SimplePrior.token_stats on the tiny golden priors (full window and a short prefix) against fp64 statistics of
    the numpy oracle transformer's logits for the same tokens and conditioning (fp16 rounding points, as the engine)"""
    from oracle.transformer_np import PriorOracle
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    m = prior.prior
    y = torch.from_numpy(fx["y"]).cuda() if "y" in fx else None
    z_conds = [torch.from_numpy(fx["z_cond"]).cuda()] if "z_cond" in fx else []
    tokens = torch.from_numpy(fx["tokens"]).cuda()
    z = prior.prior_postprocess(tokens) if prior.single_enc_dec else tokens
    if D is not None:
        z = z[:, :D].contiguous()
    k = 8
    st = prior.token_stats(z, z_conds, y, top_k=k)
    with torch.no_grad():
        x_cond, y_cond, lyric = prior.get_cond(z_conds or None, y)
        if prior.single_enc_dec:
            seq, x_cond = prior.prior_preprocess([lyric, z], [None, x_cond])
        else:
            seq = z
    from jukebox_b200.hparams import setup_hparams
    hp = setup_hparams(fx.cfg["pr_name"], dict(restore_prior="", **fx.cfg["pr_over"]))
    sd = {n: p.detach().cpu().numpy() for n, p in m.state_dict().items()}
    orc = PriorOracle(sd, m.input_dims, m.bins, m.width, m.depth, m.transformer.n_head, attn_order=hp.attn_order,
                      blocks=hp.blocks, x_cond=m.x_cond, y_cond=m.y_cond, encoder_dims=m.encoder_dims,
                      merged_decoder=not m.add_cond_after_transformer, prime_len=m.prime_len)
    xc = None if x_cond is None else x_cond.cpu().numpy()
    yc = None if y_cond is None else y_cond.cpu().numpy()
    zref = orc.logits(seq.cpu().numpy(), xc, yc, None, True, n_steps=seq.shape[1]).astype(np.float64)
    pl = seq.shape[1] - z.shape[1]
    zref = zref[:, pl:]
    n, d = z.shape
    assert st.logp.shape == (n, d) and st.entropy.shape == (n, d) and st.topk_ids.shape == (n, d, k)
    eps = TOL_PREFILL * float(np.abs(zref).max())          # the engine's logit error bound against the oracle
    lp = score_np.logprob_from_logits(zref, seq[:, pl:].cpu().numpy())
    H = stats_np.entropy_from_logits(zref)
    dlp = float(np.abs(st.logp.cpu().double().numpy() - lp).max())
    dH = float(np.abs(st.entropy.cpu().double().numpy() - H).max())
    print(f"prior_{tag} D={d}: |dlogp| {dlp:.2e}, |dH| {dH:.2e} against eps {eps:.2e}")
    assert dlp <= 2 * eps and dH <= 4 * eps
    # the ids of the CA2D over the whole sequence, and SimplePrior's mapping of them into the level's code space
    raw = m.token_stats(seq, x_cond, y_cond, top_k=k) if prior.single_enc_dec else st
    shift = prior.spaces.shift[-1] if prior.single_enc_dec else 0
    raw_ids = raw.topk_ids[:, pl:]
    assert torch.equal(raw.logp[:, pl:], st.logp) and torch.equal(raw.topk_logp[:, pl:], st.topk_logp)
    assert torch.equal(st.topk_ids, torch.where(raw_ids >= shift, raw_ids - shift, torch.full_like(raw_ids, -1)))
    assert ((st.topk_ids >= -1) & (st.topk_ids < prior.l_bins)).all()
    zr = zref.reshape(n * d, -1)
    ranked = -np.sort(-zr, axis=-1)[:, :k]
    got_z = np.take_along_axis(zr, raw_ids.cpu().numpy().reshape(n * d, k), -1)
    dz = float(np.abs(got_z - ranked).max())
    print(f"prior_{tag} D={d}: top-{k} logits at rank vs oracle {dz:.2e}, {int((st.topk_ids < 0).sum())} lyric ids")
    assert dz <= 2 * eps


def test_song_token_stats_matches_the_sampler():
    """a level of three windows (hop n_ctx / 2) drawn window by window with get_logprobs, as LevelRun draws it; then
    song_token_stats over the finished level gives each drawn code the log-probability the sampler gave it"""
    from jukebox_b200.sample import plan_windows, song_token_stats, song_windows
    fx = Fixture("prior_upsampler")
    prior = _make_prior(fx)
    n, n_ctx = 3, prior.n_ctx
    hop = n_ctx // 2
    T = 2 * n_ctx
    g = torch.Generator().manual_seed(11)
    zs = [torch.zeros(n, 0, dtype=torch.long, device="cuda"),
          torch.randint(0, prior.l_bins, (n, T // prior.cond_downsample), generator=g).cuda()]
    labels = dict(y=torch.zeros(n, 0, dtype=torch.long), info=[{}] * n)
    assert len(song_windows(T, n_ctx, hop)) == len(plan_windows(0, T, n_ctx, hop)) == 3
    lp_sampled = torch.full((n, T), float("nan"), device="cuda")
    torch.manual_seed(3)
    for win in plan_windows(0, T, n_ctx, hop):
        have = zs[0].shape[1]
        context = zs[0][:, win.start:]
        upper = prior.get_z_conds(zs, win.start, win.start + n_ctx)
        y = prior.get_y(labels, win.start)
        codes, lp = prior.sample(n, z=context, z_conds=[u.contiguous() for u in upper], y=y, fp16=True, temp=0.95,
                                 get_logprobs=True)
        new = win.start + n_ctx - have
        lp_sampled[:, have:have + new] = lp[:, -new:]
        zs[0] = torch.cat([zs[0], codes[:, -new:]], dim=1)
    assert zs[0].shape == (n, T) and bool(torch.isfinite(lp_sampled).all())
    st = song_token_stats(prior, zs, labels, 0, hop, top_k=4, max_batch_size=2)
    assert st.logp.shape == (n, T) and st.entropy.shape == (n, T) and st.topk_ids.shape == (n, T, 4)
    e = rel_err(st.logp.cpu().numpy(), lp_sampled.cpu().numpy())
    print(f"song_token_stats vs the sampler's get_logprobs over {T} codes: rel {e:.2e}")
    assert e < TOL_PREFILL
    assert bool((st.entropy > 0).all()) and bool((st.topk_logp[..., 0] >= st.logp - 1e-6).all())
    # in one piece: each window scored on its own gives the song's numbers at the positions it owns
    whole = song_token_stats(prior, zs, labels, 0, hop, top_k=4)
    assert rel_err(whole.logp.cpu().numpy(), st.logp.cpu().numpy()) < TOL_PREFILL
    for win, t0, t1 in song_windows(T, n_ctx, hop):
        upper = prior.get_z_conds(zs, win.start, win.start + n_ctx)
        one = prior.token_stats(zs[0][:, win.start:t1].contiguous(), [u.contiguous() for u in upper], None, top_k=4)
        for a, b in zip(one, whole):
            assert torch.equal(a[:, t0 - win.start:], b[:, t0:t1])


@pytest.mark.parametrize("tag", ["single_enc_dec", "upsampler"])
def test_fp32_token_stats_of_a_prefix_are_the_full_windows(tag):
    """token_stats(fp16=False) of a causal prefix of D codes: the first D positions of the fp32 full window, within the
    fp32 path's summation-order noise (tests/test_gpu_acts.py: 2e-5 of the activations' range; a log-probability moves
    by at most twice a logit's error)"""
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    y = torch.from_numpy(fx["y"]).cuda() if "y" in fx else None
    z_conds = [torch.from_numpy(fx["z_cond"]).cuda()] if "z_cond" in fx else []
    tokens = torch.from_numpy(fx["tokens"]).cuda()
    z = prior.prior_postprocess(tokens) if prior.single_enc_dec else tokens
    full = prior.token_stats(z, z_conds, y, fp16=False, top_k=4)
    D = 40
    short = prior.token_stats(z[:, :D].contiguous(), z_conds, y, fp16=False, top_k=4)
    assert short.logp.shape == (z.shape[0], D) and short.topk_ids.shape == (z.shape[0], D, 4)
    for name in ("logp", "entropy", "lse", "topk_logp"):
        a, b = getattr(short, name), getattr(full, name)[:, :D]
        d = float((a - b).abs().max())
        print(f"prior_{tag} fp32 prefix of {D}: |d {name}| {d:.2e}")
        assert d <= 4e-5 * max(1.0, float(b.abs().max())), (name, d)
