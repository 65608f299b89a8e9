"""Token scoring on the GPU: jk_xout_logprob (fused x_out + log-softmax at the target, csrc/score.cu) against the fp64
oracle over every released x_out shape; jk_sample_categorical_scored against jk_sample_categorical (same tokens) and
fp64 log-softmax; sample(get_logprobs=True) on the tiny priors, prefilled and stepped; SimplePrior.score against
z_forward's losses."""
import numpy as np
import pytest
import torch

from golden_util import Fixture
from oracle import score_np

pytestmark = pytest.mark.gpu

TOL_LOGP = 2e-5          # nats, |logp - fp64| for logits within |z| <~ 30: DESIGN.md "Scoring tokens" derives it
REL_Z = 6e-7             # beyond that: |logp - fp64| <= REL_Z * max|z| (the tensor core's in-block truncation)


def _case(W, bins, M, seed, wide=2.0):
    """activations with logits of std ~3, every fifth row `wide` times that (std 6: logits up to ~30); targets in the
    first bin, the last bin, the ragged tail bins and at random"""
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(M, W, generator=g, dtype=torch.float64)
    h[::5] *= wide
    w = torch.randn(bins, W, generator=g, dtype=torch.float64) * (3.0 / W ** 0.5)
    tg = torch.randint(0, bins, (M,), generator=g)
    tail = bins // 128 * 128
    fixed = [0, bins - 1] + ([tail, (tail + bins - 1) // 2] if tail < bins else [bins - 128, bins - 64])
    for i, v in enumerate(fixed[:M]):
        tg[i] = v
    return h.float(), w.float(), tg


@pytest.mark.parametrize("W", [1024, 1280, 1920, 2048, 4800])
def test_xout_logprob_against_fp64(W):
    from jukebox_b200.score import xout_logprob
    worst = 0.0
    for bins in (80, 1024, 2048, 2127):
        for M in (1, 127, 301):
            h, w, tg = _case(W, bins, M, seed=W + bins + M)
            want, want_lse = score_np.xout_logprob(h.double().numpy(), w.double().numpy(), tg.numpy())
            hg, wg, tgg = h.cuda(), w.cuda(), tg.cuda()
            lp, lse = xout_logprob(hg, wg, tgg, get_lse=True)
            d = float(np.abs(lp.cpu().double().numpy() - want).max())
            dl = float(np.abs(lse.cpu().double().numpy() - want_lse).max())
            worst = max(worst, d)
            assert d <= TOL_LOGP and dl <= TOL_LOGP, (W, bins, M, d, dl)
            if M == 301:
                for k in (0, 150, 300):          # a row alone gives the bits it gives in the batch
                    alone = xout_logprob(hg[k:k + 1], wg, tgg[k:k + 1])
                    assert torch.equal(alone, lp[k:k + 1]), (W, bins, k)
    print(f"xout_logprob W={W}: max |dlogp| vs fp64 {worst:.2e} nats")


@pytest.mark.parametrize("W,bins", [(1024, 80), (2048, 2127), (4800, 2127)])
def test_xout_logprob_extreme_spread(W, bins):
    """rows with logits of std 15 (|z| up to ~60): the error grows with max|z|, and stays below the fp32 SGEMM's
    (the route z_forward takes to the same numbers)"""
    from jukebox_b200.score import xout_logprob
    from jukebox_b200.transformer import f32
    h, w, tg = _case(W, bins, 301, seed=7 * W + bins, wide=5.0)
    want, want_lse = score_np.xout_logprob(h.double().numpy(), w.double().numpy(), tg.numpy())
    zmax = float(np.abs(h.double().numpy() @ w.double().numpy().T).max())
    lp, lse = xout_logprob(h.cuda(), w.cuda(), tg.cuda(), get_lse=True)
    d = float(np.abs(lp.cpu().double().numpy() - want).max())
    dl = float(np.abs(lse.cpu().double().numpy() - want_lse).max())
    sg = score_np.logsumexp(f32.linear_nk(h.cuda(), w.cuda()).cpu().double().numpy())
    ds = float(np.abs(sg - want_lse).max())
    print(f"xout_logprob W={W} bins={bins} max|z| {zmax:.0f}: |dlogp| {d:.2e}, |dlse| {dl:.2e} (fp32 SGEMM |dlse| {ds:.2e})")
    assert max(d, dl) <= REL_Z * zmax
    assert dl <= ds


def test_xout_logprob_rejects_what_the_split_cannot_hold():
    from jukebox_b200.score import xout_logprob
    h, w, tg = _case(1024, 2127, 200, seed=1)
    hg, wg, tgg = h.cuda(), w.cuda(), tg.cuda()
    bad = hg.clone()
    bad[17, 3] = 1e6
    with pytest.raises(RuntimeError, match="fp16 split"):
        xout_logprob(bad, wg, tgg)
    bad[17, 3] = float("inf")
    with pytest.raises(RuntimeError, match="fp16 split"):
        xout_logprob(bad, wg, tgg)
    wbad = wg.clone()
    wbad[5, 5] = 300.0                        # 2^8 w beyond the fp16 range
    with pytest.raises(RuntimeError, match="x_out weight"):
        xout_logprob(hg, wbad, tgg)
    tbad = tgg.clone()
    tbad[3] = 2127
    with pytest.raises(RuntimeError, match="target"):
        xout_logprob(hg, wg, tbad)
    # and the valid call after them is unaffected
    lp = xout_logprob(hg, wg, tgg)
    want, _ = score_np.xout_logprob(h.double().numpy(), w.double().numpy(), tg.numpy())
    assert float(np.abs(lp.cpu().double().numpy() - want).max()) <= TOL_LOGP


@pytest.mark.parametrize("bins,filt", [(2127, None), (2048, ("k", 40)), (2127, ("p", 0.9)), (80, None)])
def test_scored_draw_matches_the_draw_and_fp64(bins, filt):
    from jukebox_b200.transformer.ops import sample_categorical, sample_categorical_scored, filter_logits_scaled
    g = torch.Generator().manual_seed(bins)
    n, L, temp, seed = 7, 6, 0.9, 987654321
    raw = (torch.randn(n, L, bins, generator=g) * 3.0).cuda()
    raw[1] *= 8.0                                 # a wide row
    a = torch.zeros(n, L, dtype=torch.long, device="cuda")
    b = torch.zeros_like(a)
    lp = torch.full((n, L), float("nan"), device="cuda")
    for p in range(L):
        x = raw[:, p]
        if filt is None:
            sample_categorical(x, temp, seed, p, a)
            sample_categorical_scored(x, x, temp, seed, p, b, lp)
        else:
            kw = dict(top_k=filt[1], top_p=0.0) if filt[0] == "k" else dict(top_k=0, top_p=filt[1])
            f = filter_logits_scaled(x, temp, kw["top_k"], kw["top_p"])
            sample_categorical(f, 1.0, seed, p, a)
            sample_categorical_scored(f, x, 1.0, seed, p, b, lp)
    assert torch.equal(a, b)
    want = score_np.logprob_from_logits(raw.cpu().double().numpy(), b.cpu().numpy())
    d = float(np.abs(lp.cpu().double().numpy() - want).max())
    print(f"scored draw bins={bins} filter={filt}: max |dlogp| {d:.2e}")
    assert d <= 1e-5
    # logits=None scores given tokens
    lp2 = torch.full_like(lp, float("nan"))
    for p in range(L):
        sample_categorical_scored(None, raw[:, p], 1.0, 0, p, b, lp2)
    assert torch.equal(lp2, lp)


def _make_prior(fx):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae, make_prior
    c = fx.cfg
    vq = make_vqvae(setup_hparams(c["vq_name"], dict(restore_vqvae="", **c["vq_over"])), "cpu")
    prior = make_prior(setup_hparams(c["pr_name"], dict(restore_prior="", **c["pr_over"])), vq, "cpu")
    prior.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
    return prior.cuda().eval()


def _conds(prior, fx):
    """the CA2D-level conditioning of the fixture's window, as SimplePrior.sample builds it"""
    y = torch.from_numpy(fx["y"]).cuda() if "y" in fx else None
    z_conds = [torch.from_numpy(fx["z_cond"]).cuda()] if "z_cond" in fx else None
    with torch.no_grad():
        x_cond, y_cond, lyric = prior.get_cond(z_conds, y)
        if prior.single_enc_dec:
            _, x_cond = prior.prior_preprocess([lyric], [None, x_cond])
            return dict(x_cond=x_cond, y_cond=y_cond)
        return dict(x_cond=x_cond, y_cond=y_cond, encoder_kv=prior.get_encoder_kv(lyric, fp16=True, sample=True))


@pytest.mark.parametrize("stepped", [False, True])
@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_sample_get_logprobs(tag, stepped, monkeypatch):
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    m = prior.prior
    if stepped:
        monkeypatch.setenv("JK_NO_PREFILL", "1")
    m.transformer.drop_engine()
    kw = _conds(prior, fx)
    tokens = torch.from_numpy(fx["tokens"]).cuda()
    n = tokens.shape[0]
    worst = 0.0
    for primed in (False, True):
        P = tokens.shape[1] // 2
        call = (lambda **a: m.primed_sample(n, tokens[:, :P].clone(), **kw, **a)) if primed else \
               (lambda **a: m.sample(n, **kw, **a))
        for how in (dict(temp=0.9), dict(temp=0.8, top_k=20)):
            torch.manual_seed(5)
            x0 = call(fp16=True, **how)
            torch.manual_seed(5)
            x1, lp1 = call(fp16=True, get_logprobs=True, **how)
            torch.manual_seed(5)
            x2, preds, lp2 = call(fp16=True, get_preds=True, get_logprobs=True, **how)
            assert torch.equal(x0, x1) and torch.equal(x0, x2)
            want = score_np.logprob_from_logits(preds.cpu().double().numpy(), x2.cpu().numpy())
            for lp in (lp1, lp2):
                d = float(np.abs(lp.cpu().double().numpy() - want).max())
                worst = max(worst, d)
                assert d <= 1e-5, (tag, stepped, primed, how, d)
    # the fp32 loop scores through the same kernel
    torch.manual_seed(6)
    x3, preds3, lp3 = m.sample(n, **kw, fp16=False, temp=0.9, get_preds=True, get_logprobs=True, sample_tokens=9)
    want = score_np.logprob_from_logits(preds3.cpu().double().numpy(), x3.cpu().numpy())
    assert float(np.abs(lp3.cpu().double().numpy() - want).max()) <= 1e-5
    m.transformer.drop_engine()
    print(f"prior_{tag} {'stepped' if stepped else 'prefilled'}: logprobs vs log_softmax(preds) max {worst:.2e}")
    # the public call: codes and their log-likelihoods, aligned
    y = torch.from_numpy(fx["y"]).cuda() if "y" in fx else None
    z_conds = [torch.from_numpy(fx["z_cond"]).cuda()] if "z_cond" in fx else None
    torch.manual_seed(7)
    z0 = prior.sample(n, z_conds=z_conds, y=y, fp16=True, temp=0.9)
    torch.manual_seed(7)
    z1, lpz = prior.sample(n, z_conds=z_conds, y=y, fp16=True, temp=0.9, get_logprobs=True)
    assert torch.equal(z0, z1) and lpz.shape == z1.shape and bool(torch.isfinite(lpz).all()) and bool((lpz <= 0).all())


@pytest.mark.parametrize("fp16", [True, False])
@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_score_matches_z_forward(tag, fp16):
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    y = torch.from_numpy(fx["y"]).cuda() if "y" in fx else None
    z_conds = [torch.from_numpy(fx["z_cond"]).cuda()] if "z_cond" in fx else []
    tokens = torch.from_numpy(fx["tokens"]).cuda()
    z = prior.prior_postprocess(tokens) if prior.single_enc_dec else tokens
    _, metrics = prior.z_forward(z, z_conds, y, fp16=fp16)
    gen, prime = prior.score(z, z_conds, y, fp16=fp16)
    assert gen.shape == (z.shape[0],)
    rg = abs(float(gen.mean()) - float(metrics["gen_loss"])) / abs(float(metrics["gen_loss"]))
    msg = f"prior_{tag} fp16={fp16}: gen bits rel {rg:.1e}"
    assert rg <= 1e-5, msg
    if tag == "upsampler":
        assert prime is None
    else:
        rp = abs(float(prime.mean()) - float(metrics["prime_loss"])) / abs(float(metrics["prime_loss"]))
        msg += f", prime bits rel {rp:.1e}"
        assert rp <= 1e-5, msg
    print(msg)


def test_logprob_of_more_items_than_a_16_row_engine_takes():
    """20 items on a stack of 5b_lyrics' width, heads and m_attn, whose engines take at most 16 rows (jk_prior_plan at
    132 SMs: K split 1, so a 32-row activation tile does not fit in shared memory): logprob and token_stats score them
    in pieces of 16 and 4, bit for bit the items scored 16 at a time"""
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = ConditionalAutoregressive2D((64,), 256, width=4800, depth=2, heads=8, attn_order=0, blocks=8,
                                        init_scale=0.1).eval()
    assert m.items_per_prefill(20) == 16
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randint(0, 256, (20, 64), device="cuda", generator=g)
    lp = m.logprob(x)
    assert lp.shape == (20, 64) and bool(torch.isfinite(lp).all())
    assert torch.equal(lp, torch.cat([m.logprob(x[:16]), m.logprob(x[16:])]))
    st = m.token_stats(x[:, :40], top_k=4)
    for a, b0, b1 in zip(st, m.token_stats(x[:16, :40], top_k=4), m.token_stats(x[16:, :40], top_k=4)):
        assert torch.equal(a, torch.cat([b0, b1]))
    assert m.transformer._engine.max_batch == 16
