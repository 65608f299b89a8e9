"""Cost of token statistics at 1b_lyrics geometry (synthetic weights), with the card it ran on.

The x_out head over a full 16-item window (16 x 8576 positions, W 2048, 2127 bins), four routes on the same activations:
  stats k=0    jk_xout_stats: logp + entropy + lse, no logits tensor
  stats k=16   the same with the 16 most likely ids and their log-probabilities
  logprob      jk_xout_logprob: logp + lse (SimplePrior.score's head)
  composed     f32.linear_nk -> [M, bins] fp32 logits -> log_softmax -> gather + entropy + topk(16)
Every shape is warmed up first; CUDA events; the routes alternate over the rounds and the minimum is reported.

    python tools/stats_time.py [--small] [--rounds R]
"""
import contextlib
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    assert torch.cuda.is_available(), "stats_time needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(f"card: {torch.cuda.get_device_name()} | nvidia-smi: {q.stdout.strip().splitlines()[0] if q.stdout else 'n/a'}")
    small = "--small" in sys.argv
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 3
    wl = bench.SMALL if small else bench.WORKLOADS["1b_lyrics"]
    with contextlib.redirect_stdout(sys.stderr):
        prior, hps = bench.build_prior(wl)
    from jukebox_b200.score import xout_logprob, xout_stats
    from jukebox_b200.transformer import f32
    ca = prior.prior
    D, W, bins = ca.input_dims, ca.width, ca.bins
    w = ca.x_out.weight
    g = torch.Generator(device="cuda").manual_seed(0)
    n = 16
    M = n * D
    h = torch.randn(M, W, device="cuda", generator=g)
    tg = torch.randint(0, bins, (M,), device="cuda", generator=g)

    def composed():
        lp = torch.log_softmax(f32.linear_nk(h, w), -1)
        top = lp.topk(16, -1)
        return lp.gather(1, tg[:, None])[:, 0], -(lp.exp() * lp).sum(-1), top.indices, top.values

    routes = {"stats k=0": lambda: xout_stats(h, w, tg, top_k=0),
              "stats k=16": lambda: xout_stats(h, w, tg, top_k=16),
              "logprob": lambda: xout_logprob(h, w, tg),
              "composed": composed}
    # agreement of the routes on this geometry, and each against fp64 on a few rows
    st = xout_stats(h, w, tg, top_k=16)
    c = composed()
    rows = torch.arange(0, M, M // 16, device="cuda")
    z64 = h[rows].double() @ w.double().T
    lp64 = torch.log_softmax(z64, -1)
    H64 = -(lp64.exp() * lp64).sum(-1)
    eH = float((st.entropy[rows].double() - H64).abs().max())
    eHc = float((c[1][rows].double() - H64).abs().max())
    same_top = float((st.topk_ids == c[2]).all(-1).float().mean())
    print(f"M={M} W={W} bins={bins}: |dH| vs fp64 on 16 rows: fused {eH:.1e}, composed {eHc:.1e}; "
          f"top-16 ids equal to the composed route's on {same_top * 100:.2f} % of rows")
    del c, st
    for fn in routes.values():          # warm-up of every shape
        fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in routes}
    for _ in range(rounds):
        for k, fn in routes.items():
            ts[k].append(timed(fn, 3))
    for k, v in ts.items():
        print(f"head n={n} M={M} {k:11s}: {min(v):8.2f} ms (rounds {['%.2f' % x for x in v]})")
    lp = min(ts["logprob"])
    print(f"stats k=0 / logprob {min(ts['stats k=0']) / lp:.2f}x, stats k=16 / logprob {min(ts['stats k=16']) / lp:.2f}x, "
          f"composed / stats k=16 {min(ts['composed']) / min(ts['stats k=16']):.1f}x")


if __name__ == "__main__":
    main()
