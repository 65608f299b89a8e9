"""Segment-parallel upsampling on the GPU (sample_level with segments, SimplePrior.regenerate(pack=True)) on the golden
upsampler prior: without the keys, or with one segment, the level is bit for bit today's; every kept code of a greedy
segmented level is the top-1 code of its own stretch's windows (its own upper-level codes and offset); the seam pass
touches only the seam spans and keeps the candidate its scores rank first, scores that re-score through token_stats;
packed regeneration of one item is the unpacked one, every packed item's candidates begin and end with that item's own
codes, and packed items do not leak into each other.  The golden upsampler has no labels, so the per-row offset in y
is checked against a fake prior only (tests/test_segments_cpu.py).

Bound: a log-probability is z - lse, so it moves by at most twice a logit's error, 2 TOL_PREFILL max|z| (max|z| from the
fp32 path), as tests/test_gpu_regenerate.py bounds re-scored codes; a score sums D - end of them.  A greedy code drawn by
the decode step may differ from the prefill's top-1 only where the prefill's top-2 log-probabilities lie within that
bound of each other."""
import pytest
import torch

from golden_util import Fixture
from test_gpu_regenerate import _capture, _window
from test_gpu_select import _make_prior

pytestmark = pytest.mark.gpu

TOL_PREFILL = 3e-3
N, T, HOP, SEGMENTS = 2, 344, 32, 4


@pytest.fixture(scope="module")
def prior():
    return _make_prior(Fixture("prior_upsampler"))


def _song(prior, seed):
    """N items of nothing at level 0 under random codes of level 1"""
    g = torch.Generator().manual_seed(seed)
    up = torch.randint(0, prior.l_bins, (N, T // prior.cond_downsample), generator=g).cuda()
    return [torch.zeros(N, 0, dtype=torch.long, device="cuda"), up]


def _sample(prior, zs, seed, **kw):
    from jukebox_b200.hparams import Hyperparams
    from jukebox_b200.sample import sample_level
    torch.manual_seed(seed)
    return sample_level([z.clone() for z in zs], None, dict(max_batch_size=8, fp16=True, **kw), 0, prior, T, HOP,
                        Hyperparams())


def _plan(prior, seam_tokens=None):
    from jukebox_b200.sample import plan_segments
    st = prior.n_ctx // 8 if seam_tokens is None else seam_tokens
    return plan_segments(T, prior.n_ctx, HOP, SEGMENTS, prior.cond_downsample, st)


def _record_passes(monkeypatch):
    """the segment rows' codes [rows, L] after the last window, and the stitched level before the seam pass"""
    from jukebox_b200.sample import SegmentedLevel
    seen = {}
    run_window, redraw = SegmentedLevel.run_window, SegmentedLevel.redraw_seams

    def rec_window(self, codes, win, items, offsets):
        seen["codes"] = run_window(self, codes, win, items, offsets)
        return seen["codes"]

    def rec_redraw(self, plan, st):
        seen["stitched"] = self.run.zs[self.run.level].clone()
        return redraw(self, plan, st)
    monkeypatch.setattr(SegmentedLevel, "run_window", rec_window)
    monkeypatch.setattr(SegmentedLevel, "redraw_seams", rec_redraw)
    return seen


def _scale(prior, z, z_conds):
    """max|logit| of the fp32 path over the window z [1, n_ctx]"""
    seq, x_cond, y_cond, enc, _, _ = prior._condition(z, z_conds, None, True)
    with torch.no_grad():
        return float(prior.prior(seq, x_cond, y_cond, enc, fp16=False, get_preds=True)[1].abs().max())


def _own(z, rows, start, end):
    """candidate rows [K, D] with everything outside [start, end) replaced by the item's own codes z [D]"""
    K = rows.shape[0]
    return torch.cat([z[None, :start].expand(K, -1), rows[:, start:end], z[None, end:].expand(K, -1)], dim=1)


def test_absent_and_one_segment_are_todays_level(prior):
    zs = _song(prior, 1)
    ref = _sample(prior, zs, 7, temp=1.0)[0]
    for extra in (dict(segments=1), dict(segments=1, seam_tokens=5, seam_candidates=3)):
        assert torch.equal(_sample(prior, zs, 7, temp=1.0, **extra)[0], ref)


def test_greedy_segments_follow_their_own_stretch(prior, monkeypatch):
    from jukebox_b200.sample import song_windows
    zs = _song(prior, 2)
    seen = _record_passes(monkeypatch)
    out = _sample(prior, zs, 3, temp=1.0, top_k=1, segments=SEGMENTS)[0]
    plan = _plan(prior)
    S, L, ds, n_ctx = SEGMENTS, plan.length, prior.cond_downsample, prior.n_ctx
    codes = seen["codes"].view(N, S, L)
    stitched = seen["stitched"]
    span = torch.zeros(T, dtype=torch.bool, device="cuda")
    for seam in plan.seams:
        span[seam.start:seam.end] = True
    assert torch.equal(out[:, ~span], stitched[:, ~span])
    checked = exempt = exempt_differ = wrong_differ = wrong_n = 0
    for j, (s, (k0, k1)) in enumerate(zip(plan.starts, plan.kept)):
        assert torch.equal(stitched[:, k0:k1], codes[:, j, k0 - s:k1 - s])
        for win, t0, t1 in song_windows(L, n_ctx, HOP):
            o = s + win.start
            for i in range(N):
                seg = codes[i:i + 1, j, win.start:t1]
                upper = [zs[1][i:i + 1, o // ds:(o + n_ctx) // ds]]
                st = prior.token_stats(seg, upper, None, fp16=True, top_k=2)
                bound = 2 * TOL_PREFILL * _scale(prior, seg, upper)
                p = torch.arange(t0, t1, device="cuda") + s                  # positions in the level
                keep = (p >= k0) & (p < k1) & ~span[p.clamp(max=T - 1)]
                got, top = seg[0, t0 - win.start:], st.topk_ids[0, t0 - win.start:, 0]
                gap = st.topk_logp[0, t0 - win.start:, 0] - st.topk_logp[0, t0 - win.start:, 1]
                close = keep & (gap <= bound)
                bad = keep & ~close & (got != top)
                assert not bool(bad.any()), \
                    f"item {i} segment {j} window {win}: {int(bad.sum())} codes are not the top-1 of their own stretch"
                checked += int(keep.sum())
                exempt += int(close.sum())
                exempt_differ += int((close & (got != top)).sum())
                # the same codes under the stretch of the other item: what a row conditioned on the wrong stretch sees
                other = [zs[1][1 - i:2 - i, o // ds:(o + n_ctx) // ds]]
                wrong = prior.token_stats(seg, other, None, fp16=True, top_k=1).topk_ids[0, t0 - win.start:, 0]
                wrong_differ += int((keep & (got != wrong)).sum())
                wrong_n += int(keep.sum())
    print(f"greedy segments: {checked} kept codes checked, {exempt} within the top-2 bound exempted "
          f"({exempt_differ} of them differ); under another item's stretch {wrong_differ} of {wrong_n} would differ")
    assert checked > T // 2
    assert wrong_differ > 0, "the upper-level codes must move the top-1 for this check to tell stretches apart"


def test_seams_keep_their_likeliest_candidate(prior, monkeypatch):
    zs = _song(prior, 4)
    seen = _record_passes(monkeypatch)
    cands = _capture(monkeypatch)
    calls = []
    regenerate = prior.regenerate

    def rec(z, start, end, K, z_conds, y, **kw):
        out = regenerate(z, start, end, K, z_conds, y, **kw)
        calls.append((z.clone(), start, end, K, [c.clone() for c in z_conds], kw, *out))
        return out
    monkeypatch.setattr(prior, "regenerate", rec)
    K = 4
    out = _sample(prior, zs, 5, temp=1.0, segments=SEGMENTS, seam_candidates=K)[0]
    plan = _plan(prior)
    stitched = seen["stitched"]
    span = torch.zeros(T, dtype=torch.bool, device="cuda")
    for seam in plan.seams:
        span[seam.start:seam.end] = True
    assert torch.equal(out[:, ~span], stitched[:, ~span])
    pairs = [(seam, i) for seams in plan.groups().values() for seam in seams for i in range(N)]
    assert len(calls) == len(cands) and sum(c[0].shape[0] for c in calls) == len(pairs)
    m = prior.prior
    worst, r = 0.0, 0
    for (ctx, start, end, k, upper, kw, new, scores), cand in zip(calls, cands):
        assert k == K and kw["pack"] and cand.shape == (ctx.shape[0] * K, ctx.shape[1])
        D = ctx.shape[1]
        for q in range(ctx.shape[0]):
            seam, i = pairs[r]
            r += 1
            assert (start, end) == (seam.start - seam.w0, seam.end - seam.w0)
            assert torch.equal(ctx[q], stitched[i, seam.w0:seam.w1])
            rows = cand[q * K:(q + 1) * K]
            assert torch.equal(rows, _own(ctx[q], rows, start, end)), f"seam {seam} item {i} ran another item's codes"
            best = int(torch.argmax(scores[q]))
            assert bool((scores[q] <= scores[q, best]).all())
            assert torch.equal(new[q, start:end], rows[best, start:end])
            assert torch.equal(out[i, seam.start:seam.end], rows[best, start:end])
            up = [u[q:q + 1] for u in upper]
            _, x_cond, _, _, _, _ = prior._condition(ctx[q:q + 1], up, None, True)
            lp = m.token_stats(rows, x_cond.expand(K, *x_cond.shape[1:]).contiguous()).logp[:, end:].double().sum(1)
            bound = 2 * TOL_PREFILL * _scale(prior, ctx[q:q + 1], up) * (D - end)
            d = float((lp.float() - scores[q]).abs().max())
            worst = max(worst, d)
            assert d <= bound, f"seam {seam} item {i}: scores {scores[q].tolist()} vs re-scored {lp.tolist()}"
    print(f"seams: {r} redrawn in {len(calls)} packed calls, scores against re-scored candidates |d| {worst:.2e}")


def test_packed_regenerate(prior, monkeypatch):
    fx = Fixture("prior_upsampler")
    z, z_conds, y = _window(prior, fx, 4, seed=9)
    D, K = z.shape[1], 8
    start, end = D // 3, D // 3 + 6
    # one item: exactly the unpacked call
    res = []
    for pack in (False, True):
        torch.manual_seed(12)
        res.append(prior.regenerate(z[:1], start, end, K, [c[:1] for c in z_conds], y, pack=pack))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    # four items on 32 rows: every item's scores re-score on its own window
    cands = _capture(monkeypatch)
    torch.manual_seed(13)
    new, scores = prior.regenerate(z, start, end, K, z_conds, y, pack=True)
    assert len(cands) == 1 and cands[0].shape == (4 * K, D)
    m = prior.prior
    for q in range(4):
        rows = cands[0][q * K:(q + 1) * K]
        assert torch.equal(z[q, :start], new[q, :start]) and torch.equal(z[q, end:], new[q, end:])
        assert torch.equal(rows, _own(z[q], rows, start, end)), f"item {q}'s candidates ran another item's codes"
        best = int(torch.argmax(scores[q]))
        assert torch.equal(new[q, start:end], rows[best, start:end])
        up = [c[q:q + 1] for c in z_conds]
        _, x_cond, _, _, _, _ = prior._condition(z[q:q + 1], up, None, True)
        lp = m.token_stats(rows, x_cond.expand(K, *x_cond.shape[1:]).contiguous()).logp[:, end:].double().sum(1)
        bound = 2 * TOL_PREFILL * _scale(prior, z[q:q + 1], up) * (D - end)
        assert float((lp.float() - scores[q]).abs().max()) <= bound
    # one item's codes and upper-level codes changed (the first item, whose row the prime steps read first, and
    # another): the other items' candidates and scores stay
    g = torch.Generator().manual_seed(14)
    for moved in (0, 2):
        z2, zc2 = z.clone(), [c.clone() for c in z_conds]
        z2[moved] = torch.randint(0, prior.l_bins, (D,), generator=g).cuda()
        zc2[0][moved] = torch.randint(0, prior.l_bins, zc2[0][moved].shape, generator=g).cuda()
        torch.manual_seed(13)
        new2, scores2 = prior.regenerate(z2, start, end, K, zc2, y, pack=True)
        c2 = cands[-1]
        for q in set(range(4)) - {moved}:
            assert torch.equal(c2[q * K:(q + 1) * K], cands[0][q * K:(q + 1) * K]), f"item {moved} moved item {q}"
            assert torch.equal(scores2[q], scores[q]) and torch.equal(new2[q], new[q])
        assert torch.equal(c2[moved * K:(moved + 1) * K], _own(z2[moved], c2[moved * K:(moved + 1) * K], start, end))
        assert not torch.equal(c2[moved * K:(moved + 1) * K, end:], cands[0][moved * K:(moved + 1) * K, end:])
    assert len(cands) == 3
    with pytest.raises(ValueError):
        prior.regenerate(z, start, end, 9, z_conds, y, pack=True)            # 36 rows
