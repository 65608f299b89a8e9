"""Regenerating a section on the GPU (ConditionalAutoregressive2D.regenerate / SimplePrior.regenerate /
sample.regenerate_level / sample.regenerate) on the golden priors: codes outside the span are untouched, the kept
candidate is the argmax of the scores, every candidate's score is the log-likelihood of the kept codes re-scored on that
candidate's whole window (token_stats), one candidate draws what primed_sample draws, and the fp32 loop agrees.

Bound: a log-probability is z - lse, so it moves by at most twice a logit's error, 2 TOL_PREFILL max|z| (max|z| from the
fp32 path), as tests/test_gpu_select.py bounds re-scored codes; a score sums D - end of them."""
import pytest
import torch

from golden_util import Fixture
from test_gpu_select import _make_prior

pytestmark = pytest.mark.gpu

TOL_PREFILL = 3e-3


def _window(prior, fx, N, seed):
    """N rows of random codes of a whole window of this level, with the fixture's conditioning, and the sequence the
    autoregressive model reads (lyric head merged for single_enc_dec) with its conditioning"""
    g = torch.Generator().manual_seed(seed)
    y0 = torch.from_numpy(fx["y"]).cuda() if "y" in fx else None
    zc0 = [torch.from_numpy(fx["z_cond"]).cuda()] if "z_cond" in fx else []
    rows = torch.arange(N, device="cuda") % (y0.shape[0] if y0 is not None else zc0[0].shape[0] if zc0 else 1)
    y = None if y0 is None else y0[rows]
    z_conds = [torch.randint(0, prior.l_bins, c[rows].shape, generator=g).cuda() for c in zc0]
    z = torch.randint(0, prior.l_bins, (N, prior.n_ctx), generator=g).cuda()
    return z, z_conds, y


def _capture(monkeypatch):
    """the candidates' token rows [K, D] of every item, as regenerate scores them"""
    from jukebox_b200.prior.autoregressive import ConditionalAutoregressive2D
    seen = []
    orig = ConditionalAutoregressive2D._suffix_acts

    def rec(self, win, end, D):
        seen.append(win.tokens.clone())
        return orig(self, win, end, D)
    monkeypatch.setattr(ConditionalAutoregressive2D, "_suffix_acts", rec)
    return seen


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_regenerate_keeps_the_likeliest_candidate(tag, monkeypatch):
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    m = prior.prior
    N, K = 2, 6
    z, z_conds, y = _window(prior, fx, N, seed=3)
    D = z.shape[1]
    start, end = D // 3, D // 3 + max(4, D // 8)
    seen = _capture(monkeypatch)
    torch.manual_seed(4)
    z_new, scores = prior.regenerate(z, start, end, K, z_conds, y, fp16=True, temp=1.0)
    assert z_new.shape == z.shape and scores.shape == (N, K) and scores.dtype == torch.float32
    assert torch.equal(z_new[:, :start], z[:, :start]) and torch.equal(z_new[:, end:], z[:, end:])
    assert bool(torch.isfinite(scores).all())
    seq, x_cond, y_cond, enc, _, pl = prior._condition(z, z_conds, y, True)
    with torch.no_grad():
        scale = float(m(seq, x_cond, y_cond, enc, fp16=False, get_preds=True)[1].abs().max())
    bound = 2 * TOL_PREFILL * scale * (D - end)
    worst = 0.0
    for i in range(N):
        cand = seen[i]                                           # [K, pl + D] in the model's token space
        assert cand.shape == (K, pl + D) and torch.equal(cand[:, pl + end:], seq[i:i + 1, pl + end:].expand(K, -1))
        assert len({tuple(r) for r in cand[:, pl + start:pl + end].tolist()}) > 1, "the candidates differ"
        best = int(torch.argmax(scores[i]))
        assert bool((scores[i] <= scores[i, best]).all())
        kept = cand[best, pl + start:pl + end]
        if prior.single_enc_dec:         # back in this level's code space, as SimplePrior.sample returns drawn ids
            kept = (kept - prior.spaces.shift[-1]).clamp(min=0)
        assert torch.equal(z_new[i, start:end], kept)
        rep = lambda v: None if v is None else v[i:i + 1].expand(K, *v.shape[1:]).contiguous()
        lp = m.token_stats(cand, rep(x_cond), rep(y_cond), rep(enc)).logp[:, pl + end:].double().sum(1)
        d = float((lp.float() - scores[i]).abs().max())
        worst = max(worst, d)
        assert d <= bound, f"{tag} item {i}: scores {scores[i].tolist()} vs re-scored {lp.tolist()} (bound {bound:.2e})"
    print(f"prior_{tag}: scores against re-scored candidates |d| {worst:.2e} (bound {bound:.2e})")


@pytest.mark.parametrize("tag", ["single_enc_dec", "sep_enc_dec", "upsampler"])
def test_one_candidate_draws_what_primed_sample_draws(tag):
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    m = prior.prior
    z, z_conds, y = _window(prior, fx, 1, seed=5)
    seq, x_cond, y_cond, enc, _, pl = prior._condition(z, z_conds, y, True)
    D = seq.shape[1]
    start, end = pl + 7, pl + 19
    torch.manual_seed(11)
    out, scores = m.regenerate(seq, start, end, 1, x_cond, y_cond, enc, fp16=True, temp=0.9)
    torch.manual_seed(11)
    ref = m.primed_sample(1, seq[:, :start].clone(), x_cond, y_cond, enc, fp16=True, temp=0.9, sample_tokens=end)
    assert torch.equal(out[:, start:end], ref[:, start:end])
    assert torch.equal(out[:, :start], seq[:, :start]) and torch.equal(out[:, end:], seq[:, end:]) and D > end


@pytest.mark.parametrize("tag", ["single_enc_dec", "upsampler"])
def test_fp32_loop_agrees_with_fp16(tag, monkeypatch):
    fx = Fixture(f"prior_{tag}")
    prior = _make_prior(fx)
    m = prior.prior
    z, z_conds, y = _window(prior, fx, 1, seed=8)
    seq, x_cond, y_cond, enc, _, pl = prior._condition(z, z_conds, y, True)
    D, K = seq.shape[1], 4
    start, end = pl + D // 4, pl + D // 4 + 6
    seen = _capture(monkeypatch)
    out = {}
    for fp16 in (True, False):
        torch.manual_seed(2)
        out[fp16] = m.regenerate(seq, start, end, K, x_cond, y_cond, enc, fp16=fp16, temp=0.05)
    with torch.no_grad():
        scale = float(m(seq, x_cond, y_cond, enc, fp16=False, get_preds=True)[1].abs().max())
    bound = 2 * TOL_PREFILL * scale * (D - end)
    same = [c for c in range(K) if torch.equal(seen[0][c], seen[1][c])]
    assert len(same) >= K // 2, "at temperature 0.05 the two loops draw the same spans"
    d = float((out[True][1][0, same] - out[False][1][0, same]).abs().max())
    print(f"prior_{tag}: fp16 vs fp32 scores |d| {d:.2e} (bound {bound:.2e}), {len(same)} of {K} spans equal")
    assert d <= bound


def test_regenerate_level_and_song_change_only_the_span():
    """sample.regenerate over the levels a chain holds (here the upsampler's level 0 under given codes of level 1):
    each level changes only inside its scaled span, and the upper codes it reads are left as they were"""
    from jukebox_b200.hparams import Hyperparams
    from jukebox_b200.sample import regenerate
    fx = Fixture("prior_upsampler")
    prior = _make_prior(fx)
    n, n_ctx = 2, prior.n_ctx
    T = n_ctx + n_ctx // 2
    g = torch.Generator().manual_seed(21)
    zs = [torch.randint(0, prior.l_bins, (n, T), generator=g).cuda(),
          torch.randint(0, prior.l_bins, (n, T // prior.cond_downsample), generator=g).cuda()]
    labels = [dict(y=torch.zeros(n, 0, dtype=torch.long), info=[{}] * n)]
    r = prior.raw_to_tokens
    s0, e0 = T // 2, T // 2 + 9
    start, end = s0 * r + r // 2, e0 * r - r // 2           # raw samples inside codes [s0, e0)
    torch.manual_seed(1)
    new, scores = regenerate([z.clone() for z in zs], labels, [dict(fp16=True, temp=1.0, max_batch_size=16)], [prior],
                             start, end, Hyperparams(n_samples=n), n_candidates=4)
    assert torch.equal(new[1], zs[1])
    assert torch.equal(new[0][:, :s0], zs[0][:, :s0]) and torch.equal(new[0][:, e0:], zs[0][:, e0:])
    assert not torch.equal(new[0][:, s0:e0], zs[0][:, s0:e0])
    assert scores[0].shape == (n, 4)
