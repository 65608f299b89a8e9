"""Segment-parallel sampling of an upsampler level (no GPU): the plan plan_segments makes over a grid of level lengths
and geometries, and the orchestration of sample_level with segments > 1 against a fake prior that records what every
call receives and draws codes that name the row, window and position they were drawn for."""
import pytest
import torch

from jukebox_b200.hparams import Hyperparams
from jukebox_b200.sample import plan_segments, plan_windows, sample_level, song_windows

# (T, n_ctx, hop, cond_downsample, segments, seam_tokens)
GRID = [
    (330736, 8192, 4096, 4, 16, 1024),     # upsampler_level_0 at 60 s (T rounded to the top level's hop)
    (330736, 8192, 4096, 4, 40, 1024),     # the most that fit
    (82684, 8192, 4096, 4, 8, 1024),       # upsampler_level_1 at 60 s
    (264600, 8192, 4096, 4, 32, 1024),     # small_upsampler's level 0 at 60 s
    (1000, 64, 32, 4, 5, 8),
    (1004, 64, 32, 4, 15, 8),
    (997, 50, 25, 1, 7, 6),                # T, n_ctx and hop multiples of nothing in common
    (997, 50, 20, 1, 19, 6),
    (640, 64, 64, 8, 9, 8),                # hop = n_ctx (no overlap)
    (192, 64, 16, 4, 3, 3),                # segments of exactly n_ctx
    (200, 64, 16, 8, 2, 60),               # the longest seam
]


def _check_plan(T, n_ctx, hop, ds, n, st):
    plan = plan_segments(T, n_ctx, hop, n, ds, st)
    L = plan.length
    assert len(plan.starts) == n and L >= n_ctx
    assert plan.windows == tuple(plan_windows(0, L, n_ctx, hop))
    # kept ranges partition [0, T), each inside its segment
    assert plan.kept[0][0] == 0 and plan.kept[-1][1] == T
    for (a0, a1), (b0, b1) in zip(plan.kept, plan.kept[1:]):
        assert a1 == b0
    for s, (k0, k1) in zip(plan.starts, plan.kept):
        assert s <= k0 < k1 <= s + L <= T
    # starts and every window boundary on a code of the level above
    for s in plan.starts:
        assert s % ds == 0
        for w in plan.windows:
            assert (s + w.start) % ds == 0 and (s + w.start + w.sample_tokens) % ds == 0
    # seams: one per boundary, disjoint, inside their windows with a kept code after them, grouped by geometry
    assert [seam.start for seam in plan.seams] == [k0 for k0, _ in plan.kept[1:]]
    for seam, (k0, k1) in zip(plan.seams, plan.kept[1:]):
        assert seam.end - seam.start == st and seam.end < k1
        assert 0 <= seam.w0 <= seam.start and seam.end < seam.w1 <= T and seam.w1 - seam.w0 == n_ctx
        assert seam.w0 % ds == 0
    for a, b in zip(plan.seams, plan.seams[1:]):
        assert a.end <= b.start
        assert a.w1 <= b.start and a.end <= b.w0, "no seam window holds another seam's span"
    groups = plan.groups()
    assert sorted(s.start for g in groups.values() for s in g) == [s.start for s in plan.seams]
    for geom, seams in groups.items():
        assert all(seam.geometry == geom for seam in seams)
    return plan


@pytest.mark.parametrize("T, n_ctx, hop, ds, n, st", GRID)
def test_plan_segments(T, n_ctx, hop, ds, n, st):
    _check_plan(T, n_ctx, hop, ds, n, st)


@pytest.mark.parametrize("T, n_ctx, hop, ds, n, st", GRID)
def test_plan_one_segment_is_plan_windows(T, n_ctx, hop, ds, n, st):
    plan = plan_segments(T, n_ctx, hop, 1, ds, st)
    assert plan.windows == tuple(plan_windows(0, T, n_ctx, hop)) and plan.seams == ()
    assert plan.starts == (0,) and plan.kept == ((0, T),)


@pytest.mark.parametrize("T, n_ctx, hop, ds, n, st", GRID)
def test_plan_every_count_up_to_the_largest(T, n_ctx, hop, ds, n, st):
    """every count from 2 up to the largest that fits plans; one more is a ValueError that names the largest"""
    with pytest.raises(ValueError) as e:
        plan_segments(T, n_ctx, hop, T // n_ctx + 2, ds, st)
    most = int(str(e.value).rsplit("at most ", 1)[1].split()[0])
    assert most >= n
    for m in range(2, most + 1):
        if T > 10 ** 5 and m not in (2, most // 2, most):
            continue
        _check_plan(T, n_ctx, hop, ds, m, st)


def test_plan_errors():
    with pytest.raises(ValueError):
        plan_segments(1002, 64, 32, 3, 4, 8)        # T not on a code of the level above
    with pytest.raises(ValueError):
        plan_segments(1000, 64, 32, 3, 4, 64)       # seam as long as the context
    with pytest.raises(ValueError):
        plan_segments(1000, 64, 32, 0, 4, 8)
    with pytest.raises(ValueError):
        plan_segments(100, 64, 32, 2, 4, 8)         # two segments of >= 64 codes do not fit 100


# ---- orchestration against a fake prior ----------------------------------------------------------------------------
UP = 10 ** 6            # upper-level code of item i at position q: i * UP + q


class FakePrior:
    """an upsampler of n_ctx codes under codes of the level above (cond_downsample ds) with a labels row whose column 1
    is the window's offset in raw samples.  sample() draws code 10^9 item + 10^4 window offset + position: the item from
    the upper codes, the offset from the labels."""

    def __init__(self, n_ctx=64, ds=4, r=8, rows=8, x_cond=True):
        self.n_ctx, self.cond_downsample, self.raw_to_tokens, self.level = n_ctx, ds, r, 0
        self.x_cond, self.rows = x_cond, rows
        self.sampled, self.regenerated = [], []

    def get_y(self, labels, start):
        y = labels['y'].clone()
        y[:, 1] += int(start * self.raw_to_tokens)
        return y

    def get_z_conds(self, zs, start, end):
        ds = self.cond_downsample
        assert start % ds == 0 and end % ds == 0
        return [zs[1][:, start // ds:end // ds]]

    def engine_rows(self):
        return self.rows

    def guided_items(self):
        return 16

    def sample(self, n_samples, z=None, z_conds=None, y=None, **kw):
        self.sampled.append(dict(n=n_samples, z=z.clone(), up=z_conds[0].clone(), y=y.clone(), kw=kw))
        item = z_conds[0][:, :1] // UP
        off = y[:, 1:2] // self.raw_to_tokens
        out = 10 ** 9 * item + 10 ** 4 * off + torch.arange(self.n_ctx)
        out[:, :z.shape[1]] = z
        return out

    def regenerate(self, z, start, end, K, z_conds, y, pack=False, **how):
        self.regenerated.append(dict(z=z.clone(), start=start, end=end, K=K, up=z_conds[0].clone(), y=y.clone(),
                                     pack=pack, how=how))
        out = z.clone()
        out[:, start:end] = -1 - torch.arange(z.shape[0])[:, None]
        return out, torch.zeros(z.shape[0], K)


def _level(prior, N, T):
    ds = prior.cond_downsample
    zs = [torch.zeros(N, 0, dtype=torch.long),
          torch.arange(N)[:, None] * UP + torch.arange(T // ds)[None]]
    labels = dict(y=torch.zeros(N, 5, dtype=torch.long), info=[{}] * N)
    return zs, labels


def _expected_segment(prior, plan, hop, i, s):
    """the codes the fake draws for item i's segment starting at s"""
    seg = torch.empty(plan.length, dtype=torch.long)
    for win, t0, t1 in song_windows(plan.length, prior.n_ctx, hop):
        seg[t0:t1] = 10 ** 9 * i + 10 ** 4 * (s + win.start) + torch.arange(t0 - win.start, t1 - win.start)
    return seg


@pytest.mark.parametrize("N, T, n, hop, max_batch, K", [
    (1, 1000, 5, 32, 8, 2),
    (3, 1004, 15, 32, 16, 2),
    (2, 640, 9, 64, 7, 4),
    (2, 256, 2, 32, 32, 3),
])
def test_segmented_level(N, T, n, hop, max_batch, K):
    prior = FakePrior()
    zs, labels = _level(prior, N, T)
    st = 8
    kw = dict(max_batch_size=max_batch, fp16=True, temp=0.9, segments=n, seam_tokens=st, seam_candidates=K)
    out = sample_level([z.clone() for z in zs], labels, kw, 0, prior, T, hop, Hyperparams())
    plan = plan_segments(T, prior.n_ctx, hop, n, prior.cond_downsample, st)
    S, r, ds = n, prior.raw_to_tokens, prior.cond_downsample
    # every window's rows in pieces of max_batch rows, item-major, each conditioned on its own stretch
    calls = iter(prior.sampled)
    for win in plan.windows:
        got = []
        while sum(c['n'] for c in got) < N * S:
            c = next(calls)
            assert c['n'] <= max_batch and c['kw'] == dict(fp16=True, temp=0.9)
            got.append(c)
        y = torch.cat([c['y'] for c in got])
        up = torch.cat([c['up'] for c in got])
        for i in range(N):
            for j, s in enumerate(plan.starts):
                row = i * S + j
                o = s + win.start
                assert int(y[row, 1]) == o * r
                assert torch.equal(up[row], zs[1][i, o // ds:(o + prior.n_ctx) // ds])
    assert next(calls, None) is None
    # the stitched level: each segment's codes exactly in its kept range, then the seam spans redrawn
    stitched = torch.empty(N, T, dtype=torch.long)
    for i in range(N):
        for s, (k0, k1) in zip(plan.starts, plan.kept):
            stitched[i, k0:k1] = _expected_segment(prior, plan, hop, i, s)[k0 - s:k1 - s]
    z = out[0]
    assert z.shape == (N, T)
    outside = torch.ones(T, dtype=torch.bool)
    for seam in plan.seams:
        outside[seam.start:seam.end] = False
        assert bool((z[:, seam.start:seam.end] < 0).all())
    assert torch.equal(z[:, outside], stitched[:, outside])
    # the packed regeneration received every seam's window of every item, with its conditioning
    seen = []
    for c in prior.regenerated:
        assert c['pack'] and c['K'] == K and c['z'].shape[0] * K <= prior.rows
        assert c['how'] == dict(fp16=True, temp=0.9)
        for row in range(c['z'].shape[0]):
            w0 = int(c['y'][row, 1]) // r
            i = int(c['up'][row, 0]) // UP
            seam = next(sm for sm in plan.seams if sm.w0 == w0)
            assert (c['start'], c['end']) == (seam.start - w0, seam.end - w0)
            assert torch.equal(c['z'][row], stitched[i, seam.w0:seam.w1])
            assert torch.equal(c['up'][row], zs[1][i, w0 // ds:(w0 + prior.n_ctx) // ds])
            seen.append((seam.start, i))
    assert sorted(seen) == sorted((seam.start, i) for seam in plan.seams for i in range(N))


def test_one_segment_is_the_plain_level():
    prior = FakePrior()
    N, T, hop = 2, 300, 32
    zs, labels = _level(prior, N, T)
    plain = sample_level([z.clone() for z in zs], labels, dict(max_batch_size=4), 0, prior, T, hop, Hyperparams())
    calls, prior.sampled = prior.sampled, []
    one = sample_level([z.clone() for z in zs], labels, dict(max_batch_size=4, segments=1, seam_tokens=5), 0, prior, T,
                       hop, Hyperparams())
    assert torch.equal(plain[0], one[0]) and not prior.regenerated
    assert [(c['n'], c['z'].shape, c['kw']) for c in calls] == [(c['n'], c['z'].shape, c['kw']) for c in prior.sampled]


@pytest.mark.parametrize("case", ["top_level", "primed", "select", "guided", "too_many"])
def test_segmented_refusals(case):
    prior = FakePrior(x_cond=case != "top_level")
    N, T = 2, 1000
    zs, labels = _level(prior, N, T)
    kw = dict(max_batch_size=8, segments=4)
    if case == "primed":
        zs[0] = torch.zeros(N, 10, dtype=torch.long)
    if case == "select":
        kw.update(select_every=4, select_keep=1)
    if case == "guided":
        kw.update(guidance_scale=2.0, guidance_labels=labels)
    if case == "too_many":
        kw.update(segments=20)
    with pytest.raises(ValueError) as e:
        sample_level(zs, labels, kw, 0, prior, T, 32, Hyperparams())
    assert ("do not fit" if case == "too_many" else "segments > 1") in str(e.value)
    assert not prior.sampled


@pytest.mark.parametrize("entry", ["partial", "single"])
def test_single_windows_refuse_segments(entry):
    from jukebox_b200.sample import sample_partial_window, sample_single_window
    prior = FakePrior()
    zs, labels = _level(prior, 2, 1000)
    kw = dict(max_batch_size=8, segments=4)
    with pytest.raises(ValueError, match="single window"):
        if entry == "partial":
            sample_partial_window(zs, labels, kw, 0, prior, 64, Hyperparams())
        else:
            sample_single_window(zs, labels, kw, 0, prior, 0, Hyperparams())
    assert not prior.sampled
    one = sample_single_window(zs, labels, dict(kw, segments=1), 0, prior, 0, Hyperparams())
    assert one[0].shape == (2, prior.n_ctx)
