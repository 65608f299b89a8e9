"""Windowed multi-level sampling on resident priors.

Entry points keep the reference's names and argument meaning (jukebox/sample.py:17-147) because notebooks and
scripts call them: sample_partial_window, sample_single_window, sample_level, _sample, ancestral_sample,
continue_sample, upsample, primed_sample, load_codes.  The work itself is organised differently:

  * `plan_windows` is a pure function: given how many tokens a level already has, how many it needs and the
    prior's context, it lists the (start, sample_tokens) windows to run.  It is what decides the stitching, so it
    is tested on the CPU against the reference's own loop (tests/test_sample_plan_cpu.py).
  * `LevelRun` owns one level's codes / labels / sampling options and executes windows: slice the context,
    fetch the per-window conditioning from the prior, split the batch into engine-sized pieces
    (`max_batch_size`), call `prior.sample`, append the new tokens.
  * `plan_segments` / `SegmentedLevel` (sampling_kwargs key `segments`): an upsampler level drawn as many equal
    stretches on the engine's rows at once, each seam then redrawn by packed regeneration (DESIGN.md).
  * priors stay on the GPU between levels; `hps.offload_priors` restores the reference's cpu() shuffling.  At
    `max_batch_size` 32 the decode engines' arenas alone (`jk_prior_plan`, computed) are 23.5 GB for `1b_lyrics` and
    20.6 GB for each `upsampler_level_*`, 64.7 GB of an 80 GB H100 (INTEGRATION.md lists what that leaves out).

Wav / HTML / alignment output (reference :110-120) is file I/O and out of scope: `_sample` returns the codes and,
when hps.get('save_dir') is set, writes the reference's `data.pth.tar` resume format per level."""
import os
from dataclasses import dataclass

import torch as t

from .utils import dist_adapter as dist
from .utils.dist_adapter import print_once
from .utils.torch_utils import empty_cache
from .utils.sample_utils import split_batch, get_starts


@dataclass(frozen=True)
class Window:
    start: int              # first token of the context handed to the prior
    sample_tokens: int      # length of that context once the window is done (<= n_ctx)


def plan_windows(have, total_length, n_ctx, hop_length):
    """Windows that extend a level holding `have` tokens to `total_length` tokens.

    total_length >= n_ctx: full windows at get_starts(total_length, n_ctx, hop_length), each filled up to n_ctx
    (windows that are already complete are still listed: running them is a no-op).
    total_length <  n_ctx: ONE window that adds `total_length` tokens to what is there, sliding the context so
    that it never exceeds n_ctx (the reference's sample_partial_window)."""
    if total_length >= n_ctx:
        return [Window(s, n_ctx) for s in get_starts(total_length, n_ctx, hop_length)]
    if have + total_length < n_ctx:
        return [Window(0, have + total_length)]
    return [Window(have + total_length - n_ctx, n_ctx)]


def window_pieces(prior, zs, labels, level, start, end, max_batch):
    """the items of the window whose context is zs[level][:, start:end], in pieces of max_batch: (context, upper-level
    codes of the window made contiguous or None, labels or None) per piece, with the window's get_z_conds / get_y"""
    z = zs[level]
    pieces = lambda v: split_batch(v, z.shape[0], max_batch)
    upper = prior.get_z_conds(zs, start, start + prior.n_ctx)
    for ctx_i, upper_i, y_i in zip(pieces(z[:, start:end]), pieces(upper), pieces(prior.get_y(labels, start))):
        yield ctx_i, None if upper_i is None else [u.contiguous() for u in upper_i], y_i


def null_labels(prior, labels):
    """The null labels of a level's labels dict (y [N, label width] and info): for each item the same total length,
    offset and window length, unknown artist, unknown genre and no lyrics (SimplePrior.null_y) - the alternative that
    classifier-free guidance steers away from.  A prior without labels has none: ValueError."""
    y = prior.null_y(None if labels is None else labels['y'])
    info = [dict(artist="unknown", genre="unknown", lyrics="", full_tokens=[]) for _ in range(y.shape[0])]
    return dict(y=y, info=info)


class LevelRun:
    """One level of one sampling job: the codes sampled so far and what is needed to extend them.
    sampling_kwargs may hold guidance_scale and guidance_labels (guided sampling, SimplePrior.sample): a labels dict like
    `labels`, or None for null_labels(prior, labels); it is windowed as the labels are (get_y), lyrics included.
    They may hold segments (default 1), seam_tokens (default n_ctx // 8) and seam_candidates (default 4): with
    segments > 1, extend_to draws an upsampler level from nothing as that many stretches side by side on the engine's
    rows and redraws each seam (SegmentedLevel); max_batch_size then counts rows (items x segments), not items, and
    the seam pass packs up to prior.engine_rows() rows (32; 16 on 5b_lyrics) whatever max_batch_size is.  Only a whole
    level (extend_to: sample_level, _sample) is drawn in segments; sample_partial_window and sample_single_window refuse
    segments > 1."""

    def __init__(self, zs, labels, sampling_kwargs, level, prior, hps):
        self.zs, self.labels, self.level, self.prior, self.hps = zs, labels, level, prior, hps
        opts = dict(sampling_kwargs)
        opts.pop('sample_tokens', None)           # per-window, set by run_window
        self.max_batch = opts.pop('max_batch_size')
        self.segments = int(opts.pop('segments', 1))
        self.seam_tokens = opts.pop('seam_tokens', None)
        self.seam_candidates = int(opts.pop('seam_candidates', 4))
        self.guidance_labels = opts.pop('guidance_labels', None)
        if opts.get('guidance_scale') is not None:
            limit = prior.guided_items()
            if self.max_batch > limit:
                raise ValueError(f"guided sampling runs 2 engine rows per item: max_batch_size {self.max_batch} needs "
                                 f"{2 * self.max_batch} rows, at most {limit} guided items fit one engine of this model")
            if self.guidance_labels is None:
                self.guidance_labels = null_labels(prior, labels)
        elif self.guidance_labels is not None:
            raise ValueError("guidance_labels are given without a guidance_scale")
        self.opts = opts

    def have(self):
        return self.zs[self.level].shape[1]

    def one_window(self):
        """a single window is asked for: segments > 1 draws a whole level, so it is refused"""
        if self.segments > 1:
            raise ValueError(f"segments {self.segments} draws a whole level (sample_level): a single window is not cut "
                             "into segments")

    def run_window(self, win):
        prior, level = self.prior, self.level
        context = self.zs[level][:, win.start:win.start + prior.n_ctx]
        given = context.shape[1]
        missing = win.sample_tokens - given
        print_once(f"Sampling {win.sample_tokens} tokens for [{win.start},{win.start + win.sample_tokens}]. "
                   f"Conditioning on {given} tokens")
        if missing <= 0:
            return
        extra = {} if win.sample_tokens == prior.n_ctx else dict(sample_tokens=win.sample_tokens)
        selecting = self.opts.get('select_every') is not None
        guided = self.guidance_labels is not None
        alts = split_batch(prior.get_y(self.guidance_labels, win.start), self.zs[level].shape[0], self.max_batch) \
            if guided else None
        done, i0 = [], 0
        for j, (ctx_i, upper_i, y_i) in enumerate(window_pieces(prior, self.zs, self.labels, level, win.start,
                                                                win.start + prior.n_ctx, self.max_batch)):
            n = ctx_i.shape[0]
            if guided:
                extra['guidance_y'] = alts[j]
            if selecting and y_i is not None and not bool((y_i == y_i[:1]).all()):
                raise ValueError(f"keep-best selection (select_every) copies samples into other samples' rows, but items "
                                 f"{i0}..{i0 + n - 1} have different labels, which the other levels' labels cannot "
                                 "follow: give the items of a batch piece one set of labels, or sample without selection")
            out = prior.sample(n_samples=n, z=ctx_i, z_conds=upper_i, y=y_i, **self.opts, **extra)
            if selecting:
                out, ancestry = out
                self.follow(ancestry, i0)
            done.append(out)
            i0 += n
        fresh = t.cat(done, dim=0)[:, -missing:]
        self.zs[level] = t.cat([self.zs[level], fresh], dim=1)

    def follow(self, ancestry, i0):
        """rows i0 .. i0 + len(ancestry) of a window now descend from those input items: the codes of every level (this
        level's earlier windows and the upper levels' codes under them) follow their item"""
        n = ancestry.shape[0]
        for lv, z in enumerate(self.zs):
            if z.shape[0] and z.shape[1]:
                z = z.clone()
                z[i0:i0 + n] = z[i0:i0 + n][ancestry.to(z.device)]
                self.zs[lv] = z

    def extend_to(self, total_length, hop_length):
        if self.segments > 1:
            return SegmentedLevel(self).extend_to(total_length, hop_length)
        for win in plan_windows(self.have(), total_length, self.prior.n_ctx, hop_length):
            self.run_window(win)
        return self.zs


# ---- whole-song statistics ----------------------------------------------------------------------------------
def song_windows(total_length, n_ctx, hop_length):
    """(window, t0, t1) for each window of plan_windows(0, total_length, n_ctx, hop_length) that draws tokens: sampling
    a level from nothing draws tokens [t0, t1) in that window, with [window.start, t0) as its context.  The [t0, t1)
    partition [0, total_length)."""
    out, have = [], 0
    for win in plan_windows(0, total_length, n_ctx, hop_length):
        end = win.start + win.sample_tokens
        if end > have:
            out.append((win, have, end))
            have = end
    return out


def song_token_stats(prior, zs, labels, level, hop_length, fp16=True, top_k=0, max_batch_size=16):
    """Statistics of every code of a level, each scored the way sampling drew it: token t is scored in the window of
    plan_windows(0, T, n_ctx, hop_length) that drew it, conditioned on that window's labels (get_y) and upper-level
    codes (get_z_conds), with the window's earlier codes as its context.  zs: the codes of every level (zs[level]
    [N, T]); labels: this level's labels, as sample_level takes them.  Items go through the engine in pieces of
    max_batch_size, as LevelRun runs them.  Returns a score.TokenStats of [N, T] logp / entropy / lse and, with top_k,
    [N, T, top_k] topk_ids / topk_logp (SimplePrior.token_stats)."""
    from .score import TokenStats
    z = zs[level]
    N, T = z.shape
    cols = []
    for win, t0, t1 in song_windows(T, prior.n_ctx, hop_length):
        done = [prior.token_stats(ctx_i.contiguous(), upper_i, y_i, fp16=fp16, top_k=top_k)
                for ctx_i, upper_i, y_i in window_pieces(prior, zs, labels, level, win.start, t1, max_batch_size)]
        cols.append(TokenStats(*(None if v[0] is None else t.cat(v, dim=0)[:, t0 - win.start:] for v in zip(*done))))
    if not cols:
        e = t.empty(N, 0, device=z.device)
        k = t.empty(N, 0, top_k, device=z.device)
        return TokenStats(e, e.clone(), k.long() if top_k else None, k if top_k else None, e.clone())
    return TokenStats(*(None if v[0] is None else t.cat(v, dim=1) for v in zip(*cols)))


# ---- regenerating a section --------------------------------------------------------------------------------
def regen_window(T, start, end, n_ctx):
    """The window (w0, w1) of a level of T codes in which codes [start, end) are regenerated: it contains the span and
    splits the rest of the context evenly between the codes before it and the codes after it, moved inside [0, T).
    The span must be shorter than n_ctx and leave codes after it (end < T) to rank the candidates by."""
    start, end, T, n_ctx = int(start), int(end), int(T), int(n_ctx)
    if not 0 <= start < end:
        raise ValueError(f"span [{start}, {end}) is empty")
    if end >= T:
        raise ValueError(f"span [{start}, {end}) leaves no codes after it in a level of {T} codes")
    if end - start >= n_ctx:
        raise ValueError(f"span of {end - start} codes does not fit a window of {n_ctx} with a code after it")
    w0 = min(max(start - (n_ctx - (end - start)) // 2, 0), max(0, T - n_ctx))
    return w0, min(T, w0 + n_ctx)


def aligned_regen_window(T, start, end, n_ctx, ds):
    """regen_window with its start moved to a multiple of ds, where the upper-level codes under a window start
    (get_z_conds)"""
    w0, w1 = regen_window(T, start, end, n_ctx)
    if w0 % ds:
        w0 -= w0 % ds
        if min(T, w0 + n_ctx) <= end:
            w0 += ds
        w1 = min(T, w0 + n_ctx)
        assert w0 <= start and end < w1, f"no window aligned to {ds} holds [{start}, {end}) and a code after it"
    return w0, w1


def regenerate_level(zs, labels, sampling_kwargs, level, prior, start, end, hps, n_candidates=16):
    """Codes [start, end) of one level drawn again, n_candidates per item, and the candidate under which the level's
    codes after the span are likeliest kept (SimplePrior.regenerate), in the window regen_window places (its start moved
    to a code of the level above when the prior reads upper-level codes), conditioned on
    that window's labels (get_y) and upper-level codes (get_z_conds) as LevelRun conditions a window.  Items go through
    the prior in pieces of max_batch_size.  Returns (zs with zs[level] replaced, scores fp32 [N, n_candidates]: each
    candidate's log-likelihood in nats of the codes after the span in the window)."""
    opts = dict(sampling_kwargs)
    if opts.get('select_every') is not None:
        raise ValueError("keep-best selection (select_every) is not combined with regeneration")
    if opts.get('guidance_scale') is not None or opts.get('guidance_labels') is not None:
        raise ValueError("guided sampling (guidance_scale / guidance_labels) is not combined with regeneration")
    z = zs[level]
    T = z.shape[1]
    w0, w1 = aligned_regen_window(T, start, end, prior.n_ctx, prior.cond_downsample if prior.x_cond else 1)
    how = {k: opts[k] for k in ('fp16', 'temp', 'top_k', 'top_p') if k in opts}
    done, scores = [], []
    for ctx_i, upper_i, y_i in window_pieces(prior, zs, labels, level, w0, w1, opts.get('max_batch_size', T)):
        out, sc = prior.regenerate(ctx_i.contiguous(), start - w0, end - w0, n_candidates, upper_i, y_i, **how)
        done.append(out)
        scores.append(sc)
    zs = list(zs)
    z = z.clone()
    z[:, start:end] = t.cat(done, dim=0)[:, start - w0:end - w0].to(z.device)
    zs[level] = z
    return zs, t.cat(scores, dim=0)


def regenerate(zs, labels, sampling_kwargs, priors, start, end, hps, n_candidates=16):
    """Regenerate the section [start, end) of raw audio samples of every level, from the top level down: each level's
    span is [start, end) in its codes (start // raw_to_tokens up to end rounded up), and each level below the top is
    drawn under the new codes above it and ranked by its own codes after the span (regenerate_level).  labels and
    sampling_kwargs per level, as _sample takes them.  Returns (zs, {level: scores [N, n_candidates]})."""
    scores = {}
    for level in sorted(range(len(priors)), reverse=True):
        prior = priors[level]
        r = prior.raw_to_tokens
        zs, scores[level] = regenerate_level(zs, labels[level], sampling_kwargs[level], level, prior, int(start) // r,
                                             -(-int(end) // r), hps, n_candidates)
    return zs, scores


# ---- segment-parallel sampling of an upsampler level ---------------------------------------------------------
@dataclass(frozen=True)
class Seam:
    start: int              # first code redrawn: a boundary between two kept ranges
    end: int                # end of the redrawn span
    w0: int                 # the window [w0, w1) of the level it is redrawn in (aligned_regen_window)
    w1: int

    @property
    def geometry(self):
        """(window length, offset of the span in it): seams of one geometry run packed on one engine window"""
        return self.w1 - self.w0, self.start - self.w0


@dataclass(frozen=True)
class SegmentPlan:
    length: int             # L: codes of every segment
    starts: tuple           # s_j: first code of segment j in the level
    windows: tuple          # the windows every segment runs, from its own start: plan_windows(0, L, ...)
    kept: tuple             # (k_j, k_j+1): the codes of the level segment j supplies; they partition [0, T)
    seams: tuple            # a Seam at every k_j, j >= 1

    def groups(self):
        """{geometry: [Seam, ...]}"""
        out = {}
        for seam in self.seams:
            out.setdefault(seam.geometry, []).append(seam)
        return out


def _segment_length(T, n, n_ctx, ds, seam_tokens):
    """the length L of n segments of a level of T codes (T / n rounded up to a multiple of ds), or None when they do not
    fit: L < n_ctx, or the last kept range too short to hold a seam span and a code after it"""
    L = -(-T // n)
    L = -(-L // ds) * ds
    return L if L >= n_ctx and T - (n - 1) * L > seam_tokens else None


def plan_segments(T, n_ctx, hop_length, n_segments, cond_downsample, seam_tokens):
    """A level of T codes drawn as n_segments stretches side by side.  Every segment has the same length L >= n_ctx and
    runs the same windows plan_windows(0, L, n_ctx, hop_length) from its own start, so that all of them stand at one
    position of the engine.  Segment j starts at s_j = j L (the last at T - L, so that it ends at T) and supplies the
    codes [k_j, k_j+1) = [j L, (j + 1) L) (the last [(n - 1) L, T): its leading overlap with the segment before is
    dropped).  Starts and windows are multiples of cond_downsample (get_z_conds).  At every k_j, j >= 1, a Seam: its span
    [k_j, k_j + seam_tokens) is drawn again in the window aligned_regen_window places, which holds kept codes after it.
    n_segments 1: the windows of plan_windows(0, T, ...) and no seams.  ValueError when the count does not fit."""
    T, n_ctx, hop, n, st = int(T), int(n_ctx), int(hop_length), int(n_segments), int(seam_tokens)
    ds = int(cond_downsample or 1)
    if n < 1:
        raise ValueError(f"segments {n} must be >= 1")
    if n == 1:
        return SegmentPlan(T, (0,), tuple(plan_windows(0, T, n_ctx, hop)), ((0, T),), ())
    if T % ds or n_ctx % ds or hop % ds:
        raise ValueError(f"segments start on codes of the level above: T {T}, n_ctx {n_ctx} and hop {hop} must be "
                         f"multiples of {ds}")
    if not 0 < st < n_ctx:
        raise ValueError(f"seam_tokens {st} outside [1, {n_ctx})")
    L = _segment_length(T, n, n_ctx, ds, st)
    if L is None:
        most = max([m for m in range(2, T // n_ctx + 2) if _segment_length(T, m, n_ctx, ds, st)], default=1)
        raise ValueError(f"{n} segments of a level of {T} codes do not fit: each needs >= n_ctx {n_ctx} codes and the "
                         f"last a seam of {st} codes with a code after it; at most {most} fit")
    bounds = [j * L for j in range(n)] + [T]
    seams = []
    for k in bounds[1:-1]:
        w0, w1 = aligned_regen_window(T, k, k + st, n_ctx, ds)
        seams.append(Seam(k, k + st, w0, w1))
    return SegmentPlan(L, tuple(bounds[:n - 1]) + (T - L,), tuple(plan_windows(0, L, n_ctx, hop)),
                       tuple(zip(bounds[:-1], bounds[1:])), tuple(seams))


def row_conditioning(prior, zs, labels, items, starts):
    """the upper-level codes (a list, or None) and label rows (or None) of engine rows that each read item items[r] in
    the window of this level that starts at starts[r] (get_z_conds / get_y of that window)"""
    per_start, ups, ys = {}, [], []
    for i, s in zip(items, starts):
        if s not in per_start:
            per_start[s] = prior.get_z_conds(zs, s, s + prior.n_ctx), prior.get_y(labels, s)
        up, y = per_start[s]
        ups.append(None if up is None else [u[i] for u in up])
        ys.append(None if y is None else y[i])
    up = None if ups[0] is None else [t.stack([u[k] for u in ups]) for k in range(len(ups[0]))]
    return up, (None if ys[0] is None else t.stack(ys))


class SegmentedLevel:
    """A LevelRun with segments > 1: the level is drawn from nothing as plan_segments' stretches.  Rows are items x
    segments, item-major (row i S + j: item i, segment j); in every window of the shared plan each row reads its own
    context, the upper-level codes under its own stretch and labels at its own offset (get_z_conds / get_y at
    s_j + window start), and the rows run through prior.sample in pieces of max_batch_size rows.  The kept ranges are
    stitched into zs[level], then every seam is redrawn given the codes on both sides of it: seam_candidates draws of its
    span, the one under which the kept codes after it are likeliest is kept (SimplePrior.regenerate, packed: seams of one
    geometry x items in pieces of the engine's rows).  No seam window holds another seam's span, so the order of the
    seams does not matter."""

    def __init__(self, run):
        prior = run.prior
        if not prior.x_cond:
            raise ValueError("segments > 1 needs an upsampler: the top level has no upper-level codes to carry the "
                             "song's structure across its stretches")
        if run.have():
            raise ValueError(f"segments > 1 draws a level from nothing, but level {run.level} already holds "
                             f"{run.have()} codes: the stretches could not share one engine position with them")
        if run.opts.get('select_every') is not None:
            raise ValueError("keep-best selection (select_every) is not combined with segments > 1")
        if run.guidance_labels is not None or run.opts.get('guidance_scale') is not None:
            raise ValueError("guided sampling (guidance_scale / guidance_labels) is not combined with segments > 1")
        self.run = run

    def extend_to(self, total_length, hop_length):
        run, prior = self.run, self.run.prior
        zs, level = run.zs, run.level
        N = zs[level].shape[0]
        st = prior.n_ctx // 8 if run.seam_tokens is None else int(run.seam_tokens)
        plan = plan_segments(total_length, prior.n_ctx, hop_length, run.segments, prior.cond_downsample, st)
        S, L = len(plan.starts), plan.length
        items = [i for i in range(N) for _ in range(S)]
        offsets = [s for _ in range(N) for s in plan.starts]
        codes = zs[level].new_zeros(N * S, 0)
        for win in plan.windows:
            codes = self.run_window(codes, win, items, offsets)
        codes = codes.view(N, S, L)
        zs[level] = t.cat([codes[:, j, k0 - s:k1 - s] for j, (s, (k0, k1)) in enumerate(zip(plan.starts, plan.kept))],
                          dim=1)
        self.redraw_seams(plan, st)
        return zs

    def run_window(self, codes, win, items, offsets):
        """codes [rows, have]: every row's stretch so far, extended by window win (from each row's own start)"""
        run, prior = self.run, self.run.prior
        context = codes[:, win.start:win.start + prior.n_ctx]
        missing = win.sample_tokens - context.shape[1]
        print_once(f"Sampling {win.sample_tokens} tokens for [{win.start},{win.start + win.sample_tokens}] of "
                   f"{codes.shape[0]} segment rows. Conditioning on {context.shape[1]} tokens")
        if missing <= 0:
            return codes
        extra = {} if win.sample_tokens == prior.n_ctx else dict(sample_tokens=win.sample_tokens)
        up, y = row_conditioning(prior, run.zs, run.labels, items, [s + win.start for s in offsets])
        part = lambda v, r: None if v is None else v[r:r + run.max_batch]
        done = []
        for r in range(0, codes.shape[0], run.max_batch):
            ctx = context[r:r + run.max_batch]
            done.append(prior.sample(n_samples=ctx.shape[0], z=ctx, z_conds=None if up is None else
                                     [u[r:r + run.max_batch].contiguous() for u in up], y=part(y, r),
                                     **run.opts, **extra))
        return t.cat([codes, t.cat(done, dim=0)[:, -missing:]], dim=1)

    def redraw_seams(self, plan, seam_tokens):
        run, prior = self.run, self.run.prior
        z = run.zs[run.level]
        K = run.seam_candidates
        how = {k: run.opts[k] for k in ('fp16', 'temp', 'top_k', 'top_p') if k in run.opts}
        per_call = max(1, prior.engine_rows() // K)
        for (_, off), seams in plan.groups().items():
            pairs = [(seam, i) for seam in seams for i in range(z.shape[0])]
            for p0 in range(0, len(pairs), per_call):
                piece = pairs[p0:p0 + per_call]
                ctx = t.stack([z[i, seam.w0:seam.w1] for seam, i in piece])
                up, y = row_conditioning(prior, run.zs, run.labels, [i for _, i in piece], [seam.w0 for seam, _ in piece])
                out, _ = prior.regenerate(ctx, off, off + seam_tokens, K, up, y, pack=True, **how)
                for r, (seam, i) in enumerate(piece):
                    z[i, seam.start:seam.end] = out[r, off:off + seam_tokens].to(z.device)


# ---- the reference's entry points -------------------------------------------------------------------------
def sample_partial_window(zs, labels, sampling_kwargs, level, prior, tokens_to_sample, hps):
    """`tokens_to_sample` new tokens at `level`, the context sliding once it is full"""
    run = LevelRun(zs, labels, sampling_kwargs, level, prior, hps)
    run.one_window()
    have = run.have()
    if have + tokens_to_sample < prior.n_ctx:
        win = Window(0, have + tokens_to_sample)
    else:
        win = Window(have + tokens_to_sample - prior.n_ctx, prior.n_ctx)
    run.run_window(win)
    return zs


def sample_single_window(zs, labels, sampling_kwargs, level, prior, start, hps):
    """the window of prior.n_ctx tokens that starts at `start`; tokens already there are the prime"""
    run = LevelRun(zs, labels, sampling_kwargs, level, prior, hps)
    run.one_window()
    run.run_window(Window(start, sampling_kwargs.get('sample_tokens', prior.n_ctx)))
    return zs


def sample_level(zs, labels, sampling_kwargs, level, prior, total_length, hop_length, hps):
    print_once(f"Sampling level {level}")
    return LevelRun(zs, labels, sampling_kwargs, level, prior, hps).extend_to(total_length, hop_length)


def _on_gpu(module):
    return all(p.is_cuda for p in module.parameters())


def _sample(zs, labels, sampling_kwargs, priors, sample_levels, hps):
    audio = {}
    for level in sorted(sample_levels, reverse=True):        # coarsest level first
        prior = priors[level]
        if not _on_gpu(prior):                               # a resident prior keeps its packed decode engine
            prior.cuda()
        assert hps.sample_length % prior.raw_to_tokens == 0, \
            f"Expected sample_length {hps.sample_length} to be multiple of {prior.raw_to_tokens}"
        tokens_needed = hps.sample_length // prior.raw_to_tokens
        hop = int(hps.hop_fraction[level] * prior.n_ctx)
        zs = sample_level(zs, labels[level], sampling_kwargs[level], level, prior, tokens_needed, hop, hps)
        if hps.get('offload_priors', False):      # the reference always did (16 GB cards); 80 GB keeps them
            prior.cpu()
            empty_cache()
        audio[level] = prior.decode(zs[level:], start_level=level, bs_chunks=zs[level].shape[0])
        out_dir = hps.get('save_dir', None)
        if out_dir:
            save_level(out_dir, level, zs, labels, sampling_kwargs, audio[level])
    hps['_last_audio'] = audio
    return zs


def save_level(save_dir, level, zs, labels, sampling_kwargs, x):
    """the reference's resume file (sample.py:116): {zs, labels, sampling_kwargs, x} per level"""
    root = f"{save_dir}_rank_{dist.get_rank()}" if dist.get_world_size() > 1 else save_dir
    logdir = os.path.join(root, f"level_{level}")
    os.makedirs(logdir, exist_ok=True)
    t.save(dict(zs=zs, labels=labels, sampling_kwargs=sampling_kwargs, x=x), os.path.join(logdir, "data.pth.tar"))
    return logdir


def _all_levels(priors):
    return list(range(len(priors)))


def ancestral_sample(labels, sampling_kwargs, priors, hps):
    empty = [t.zeros(hps.n_samples, 0, dtype=t.long, device='cuda') for _ in priors]
    return _sample(empty, labels, sampling_kwargs, priors, _all_levels(priors), hps)


def continue_sample(zs, labels, sampling_kwargs, priors, hps):
    return _sample(zs, labels, sampling_kwargs, priors, _all_levels(priors), hps)


def upsample(zs, labels, sampling_kwargs, priors, hps):
    return _sample(zs, labels, sampling_kwargs, priors, _all_levels(priors)[:-1], hps)


def primed_sample(x, labels, sampling_kwargs, priors, hps):
    zs = priors[-1].encode(x, start_level=0, end_level=len(priors), bs_chunks=x.shape[0])
    return _sample(zs, labels, sampling_kwargs, priors, _all_levels(priors), hps)


def load_codes(codes_file, duration, priors, hps):
    """codes of a previous run (`data.pth.tar`), optionally cut to `duration` raw samples"""
    stored = t.load(codes_file, map_location='cpu', weights_only=False)['zs']
    assert stored[-1].shape[0] == hps.n_samples, f"Expected bs = {hps.n_samples}, got {stored[-1].shape[0]}"
    keep = [z.shape[1] for z in stored]
    if duration is not None:
        top = priors[-1].raw_to_tokens
        assert duration % top == 0, f"duration {duration} is not a multiple of {top}"
        assert duration // top <= stored[-1].shape[1]
        keep = [duration // prior.raw_to_tokens for prior in priors]
    return [z[:, :k].cuda() for z, k in zip(stored, keep)]
