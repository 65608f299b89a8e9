"""Cost of regenerating a section at 1b_lyrics geometry (synthetic weights), with the card it ran on.

For 16 rows standing at position t0 in {1024, 4096, 7680} (moved back so that t0 + m fits the window), and a suffix of
m in {256, 1024} kept codes:
  continue  - the continuation prefill of the m positions (jk_prior_prefill on an engine at t0);
  step      - the same m positions stepped (m decode launches);
  prefill   - one prefill of [0, t0 + m) from the head of the window (what scoring the whole window again costs);
and one whole ConditionalAutoregressive2D.regenerate call on the prior's token sequence: 16 candidates of the 128 codes
before t0, ranked by the m codes after them (one-row prime prefill of t0 - 128 positions, broadcast, 128 sampled steps,
the continuation prefill, the scoring head).
The three routes alternate within every round; every shape runs once before the timed rounds; CUDA events; min /
median over the rounds.

    python tools/regen_time.py [--small] [--rounds R]
"""
import contextlib
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def fmt(ts):
    return f"{min(ts):9.2f} / {statistics.median(ts):9.2f} ms"


def main():
    assert torch.cuda.is_available(), "regen_time needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(f"card: {torch.cuda.get_device_name()} | nvidia-smi: {q.stdout.strip().splitlines()[0] if q.stdout else 'n/a'}")
    small = "--small" in sys.argv
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 3
    wl = bench.SMALL if small else bench.WORKLOADS["1b_lyrics"]
    with contextlib.redirect_stdout(sys.stderr):
        prior, _ = bench.build_prior(wl)
    ca = prior.prior
    D, W, n = ca.input_dims, ca.width, 16
    eng = ca._engine(n)
    cap = eng.prefill_capacity
    g = torch.Generator(device="cuda").manual_seed(0)
    toks = torch.randint(0, ca.bins, (n, D), device="cuda", generator=g)
    yc = torch.randn(n, W, device="cuda", generator=g) * 0.1 if ca.y_cond else None
    xc = torch.randn(n, D, W, device="cuda", generator=g) * 0.01 if ca.x_cond else None
    print(f"1b_lyrics geometry: {ca.depth} layers, width {W}, {D} positions, prefill capacity {cap}, {n} rows")
    small_ctx = D < 2048
    span = 8 if small_ctx else 128
    for t0_want in ((16, 64, 200) if small_ctx else (1024, 4096, 7680)):
        for m in ((8, 32) if small_ctx else (256, 1024)):
            t0 = min(t0_want, D - m)

            def at_t0():                # the rows at position t0 (not timed)
                eng.reset(0)
                eng.prefill(n, t0, tokens=toks, y_cond=yc, x_cond=xc)
                torch.cuda.synchronize()

            def cont():
                eng.prefill(n, m, tokens=toks, x_cond=xc)

            def step():
                for _ in range(m):
                    eng.step(n, tokens=toks, y_cond=yc, x_cond=xc)

            def whole():
                eng.reset(0)
                eng.prefill(n, t0 + m, tokens=toks, y_cond=yc, x_cond=xc)

            routes = {"continue": (at_t0, cont), "step": (at_t0, step)}
            if t0 + m <= cap:
                routes["prefill [0, t0+m)"] = (None, whole)
            for setup, fn in routes.values():      # warm-up of every shape
                if setup:
                    setup()
                timed(fn)
            res = {k: [] for k in routes}
            for _ in range(rounds):
                for k, (setup, fn) in routes.items():
                    if setup:
                        setup()
                    res[k].append(timed(fn))
            print(f"t0 {t0}, m {m} (min / median of {rounds}):")
            for k, ts in res.items():
                print(f"  {k:18s}: {fmt(ts)}  ({min(ts) / m * 1e3:8.1f} us per position)")
            print(f"  continue vs step: x{min(res['step']) / min(res['continue']):.1f}")
            # one whole regenerate call: 16 candidates of [t0 - span, t0), ranked by [t0, t0 + m)
            x = toks[:1, :t0 + m].clone()
            xc1 = None if xc is None else xc[:1]
            yc1 = None if yc is None else yc[:1, None]
            run = lambda: ca.regenerate(x, t0 - span, t0, n, xc1, yc1, None, fp16=True, temp=1.0)
            timed(run)
            ts = [timed(run) for _ in range(rounds)]
            print(f"  regenerate, {n} candidates of {span} codes: {fmt(ts)}")


if __name__ == "__main__":
    main()
