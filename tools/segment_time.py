"""Wall time of one upsampler level of a 60 s song drawn plainly (segments 1) and as segments on the engine's idle rows,
at small_upsampler and upsampler_level_0 geometry with synthetic weights (bench.synth_fill), with the card it ran on.

T = 330 736 codes for both: level 0 of the three-level VQ-VAE at 60 s of 44.1 kHz, cut to a multiple of the top level's
128 samples as the reference's sample length is.  small_upsampler stands in for a cheaper step at the same length.  For
N = 1 and 3 items: segments 1 (N rows), and the largest count S with N S <= 16 and N S <= 32 rows (max_batch_size N S).

Printed separately:
  step      - the decode step + draw of SamplingWindow.advance at 1, 3, 16 and 32 rows, 256 positions from position
              n_ctx / 2 (median of --rounds);
  segment   - the segment pass (SegmentedLevel.run_window over the plan's windows); segments 1: LevelRun.run_window;
  seam      - the seam pass (SegmentedLevel.redraw_seams: seam_candidates 4, seam_tokens n_ctx // 8), always run whole;
  level     - segment + seam.
Time bound: only the first --windows windows of each pass run (default 2: the ancestral one and one primed by half a
window); the rest of the pass is extrapolated from the second measured window's time per drawn code, times the codes
the remaining windows draw.  Lines say "extrapolated" when that happened and "measured" when every window ran.
CUDA events; every shape runs once before it is timed.

    python tools/segment_time.py [--priors small_upsampler,upsampler_level_0] [--items 1,3] [--windows 2] [--rounds 3]
"""
import argparse
import contextlib
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import hps_pair, make_labels, synth_fill  # noqa: E402

T_LEVEL0 = 2646000 // 128 * 128 // 8
PRIORS = {
    "small_upsampler": ("small_vqvae", 8192 * 32, dict(labels=False, level=0, levels=2)),
    "upsampler_level_0": ("vqvae", 8192 * 8, dict()),
}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def build(name, seed=0):
    from jukebox_b200.make_models import make_vqvae, make_prior
    vq, length, over = PRIORS[name]
    vq_h, pr_h = hps_pair(dict(vq=(vq, dict(sample_length=length)), prior=(name, over)))
    with torch.device("cuda"), contextlib.redirect_stdout(sys.stderr):
        prior = make_prior(pr_h, make_vqvae(vq_h, "cuda"), "cuda")
    synth_fill(prior, seed)
    return prior.eval(), pr_h


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3, out


def step_time(prior, n, m=256, rounds=3):
    """seconds per position of SamplingWindow.advance on n rows at positions [n_ctx / 2, n_ctx / 2 + m)"""
    from jukebox_b200.prior.autoregressive import SamplingWindow
    ca = prior.prior
    D, W = ca.input_dims, ca.width
    g = torch.Generator(device="cuda").manual_seed(n)
    P = D // 2
    prime = torch.randint(0, ca.bins, (n, P), device="cuda", generator=g)
    xc = torch.randn(n, D, W, device="cuda", generator=g) * 0.01
    yc = torch.randn(n, 1, W, device="cuda", generator=g) * 0.1 if ca.y_cond else None
    ts = []
    for r in range(rounds + 1):
        win = SamplingWindow(ca, n, prime, xc, yc, None, True, 1.0, 0, 0.0, False, None)
        dt, _ = timed(lambda: win.advance(P + m))
        ca.transformer.del_cache()
        if r:
            ts.append(dt / m)
    return statistics.median(ts)


def level_time(prior, labels, N, S, hop, windows):
    """(segment pass seconds, seam pass seconds or None, measured whole?) of one level of T_LEVEL0 codes"""
    from jukebox_b200.hparams import Hyperparams
    from jukebox_b200.sample import LevelRun, SegmentedLevel, plan_segments, song_windows
    T, n_ctx, ds = T_LEVEL0, prior.n_ctx, prior.cond_downsample
    g = torch.Generator().manual_seed(S)
    zs = [torch.zeros(N, 0, dtype=torch.long, device="cuda"),
          torch.randint(0, prior.l_bins, (N, T // ds), generator=g).cuda()]
    kw = dict(max_batch_size=N * S, fp16=True, temp=1.0, segments=S)
    run = LevelRun(zs, labels, kw, 0, prior, Hyperparams())
    st = n_ctx // 8
    plan = plan_segments(T, n_ctx, hop, S, ds, st)
    drawn = [t1 - t0 for _, t0, t1 in song_windows(plan.length, n_ctx, hop)]
    if S == 1:
        step = lambda win, _codes: run.run_window(win)
    else:
        seg = SegmentedLevel(run)
        items = [i for i in range(N) for _ in range(S)]
        offsets = [s for _ in range(N) for s in plan.starts]
        step = lambda win, codes: seg.run_window(codes, win, items, offsets)
    # warm-up of the windows' shapes on N S rows: an ancestral head, and a window primed by hop codes
    R = N * S
    upper = [zs[1][:1, :n_ctx // ds].expand(R, -1).contiguous()]
    y = None if labels is None else prior.get_y(labels, 0)[:1].expand(R, -1).contiguous()
    prior.sample(R, z=None, z_conds=upper, y=y, fp16=True, sample_tokens=64)
    prior.sample(R, z=torch.randint(0, prior.l_bins, (R, hop), generator=g).cuda(), z_conds=upper, y=y, fp16=True,
                 sample_tokens=hop + 64)
    codes = zs[0].new_zeros(N * S, 0)
    ts = []
    for win in plan.windows[:windows]:
        dt, codes = timed(lambda: step(win, codes))
        ts.append(dt)
    whole = len(ts) == len(drawn)
    seg_s = sum(ts) if whole else sum(ts) + ts[-1] / drawn[len(ts) - 1] * sum(drawn[len(ts):])
    if S == 1:
        return seg_s, None, whole
    run.zs[0] = torch.randint(0, prior.l_bins, (N, T), generator=g).cuda()       # a stitched level to redraw
    seg.redraw_seams(plan, st)                                                    # warm-up
    seam_s, _ = timed(lambda: seg.redraw_seams(plan, st))
    return seg_s, seam_s, whole


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--priors", default="small_upsampler,upsampler_level_0")
    ap.add_argument("--items", default="1,3")
    ap.add_argument("--windows", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "segment_time needs a GPU"
    print(f"card: {torch.cuda.get_device_name()} | nvidia-smi name, power limit, max SM clock: {gpu_info()}")
    from jukebox_b200.sample import plan_segments
    for name in a.priors.split(","):
        prior, pr_h = build(name)
        hop = int(0.5 * prior.n_ctx)
        print(f"{name}: width {prior.prior.width}, {prior.prior.depth} layers, n_ctx {prior.n_ctx}, hop {hop}, "
              f"T {T_LEVEL0} codes (60 s at level 0)")
        with contextlib.redirect_stdout(sys.stderr):
            for n in (1, 3, 16, 32):
                step_time(prior, n, m=16, rounds=1)                  # warm-up of every row count
            steps = {n: step_time(prior, n, rounds=a.rounds) for n in (1, 3, 16, 32)}
        print("  step: " + ", ".join(f"{n} rows {s * 1e3:.3f} ms" for n, s in steps.items()))
        for N in (int(v) for v in a.items.split(",")):
            y = make_labels(prior, pr_h, N, 0)
            labels = None if y is None else dict(y=y.cuda(), info=[dict(full_tokens=[])] * N)
            most = 1
            for m in range(2, T_LEVEL0 // prior.n_ctx + 2):
                with contextlib.suppress(ValueError):
                    plan_segments(T_LEVEL0, prior.n_ctx, hop, m, prior.cond_downsample, prior.n_ctx // 8)
                    most = m
            counts = [1] + sorted({min(most, rows // N) for rows in (16, 32)})
            base = None
            for S in counts:
                with contextlib.redirect_stdout(sys.stderr):
                    seg_s, seam_s, whole = level_time(prior, labels, N, S, hop, a.windows)
                total = seg_s + (seam_s or 0.0)
                base = base or total
                how = "measured" if whole else f"first {a.windows} windows measured, the rest extrapolated"
                seam = "" if seam_s is None else f", seam pass {seam_s:8.2f} s (measured)"
                print(f"  N {N}, segments {S:2d} ({N * S:2d} rows): level {total:8.1f} s (x{base / total:5.2f}), "
                      f"segment pass {seg_s:8.1f} s ({how}){seam}")
        del prior
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
