"""Cost of sample selection (jk_prior_select) at 1b_lyrics geometry (synthetic weights), with the card it ran on.

1. jk_prior_select on engines of 16 and 32 rows: a broadcast of row 0 (every other row overwritten, nothing stashed)
   and the worst case, a reversal of every row (every row stashed, then every row copied), against the least time
   their bytes take at the H100 SXM data sheet's 3.35 TB/s.  The K / V caches are copied whole, so the time does not
   depend on the position.
2. One prime of 4096 positions continued in 16 rows: prefilled on one row and broadcast (prefill(1) + select), against
   prefilling 16 copies of it (prefill(16)), the cost a one-row prime saves.
Cases alternate within every round; every shape runs once before the timed rounds; min / median over the rounds.

    python tools/select_time.py [--small] [--rounds R]
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

HBM_TBS = 3.35          # H100 SXM data sheet, HBM3


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def rounds_of(cases, rounds, reps):
    """{name: [ms per call of each round]}, the cases alternating within a round, after one warm-up call each"""
    for fn in cases.values():
        fn()
    torch.cuda.synchronize()
    out = {k: [] for k in cases}
    for _ in range(rounds):
        for k, fn in cases.items():
            out[k].append(timed(fn, reps))
    return out


def fmt(ts):
    return f"{min(ts):.3f} / {statistics.median(ts):.3f} ms"


def main():
    assert torch.cuda.is_available(), "select_time needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(f"card: {torch.cuda.get_device_name()} | nvidia-smi: {q.stdout.strip().splitlines()[0] if q.stdout else 'n/a'}")
    small = "--small" in sys.argv
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 7
    wl = bench.SMALL if small else bench.WORKLOADS["1b_lyrics"]
    with contextlib.redirect_stdout(sys.stderr):
        prior, _ = bench.build_prior(wl)
    ca = prior.prior
    tr = ca.transformer
    D, W = ca.input_dims, ca.width

    # ---- 1. the copies ----
    for n in (16, 32):
        tr.drop_engine()
        torch.cuda.empty_cache()
        eng = ca._engine(n)
        eng.reset(0)
        bcast, rev = [0] * n, list(range(n - 1, -1, -1))
        pb, pr = eng.select_plan(bcast), eng.select_plan(rev)
        res = rounds_of({"broadcast": lambda: eng.select(bcast), "reversal": lambda: eng.select(rev)}, rounds, 10)
        print(f"select, {n} rows, one row's K / V {pb.row_bytes / 1e6:.1f} MB over {ca.depth} layers:")
        for name, p in (("broadcast", pb), ("reversal", pr)):
            bound = p.bytes_moved / (HBM_TBS * 1e12) * 1e3
            ts = res[name]
            print(f"  {name:9s}: {fmt(ts)} (min / median of {rounds}), {p.bytes_moved / 1e9:.2f} GB moved "
                  f"(stash {p.n_stash} rows, {p.workspace_bytes / 1e9:.2f} GB workspace), {p.bytes_moved / min(ts) / 1e6:.0f} GB/s "
                  f"= {bound / min(ts) * 100:.0f} % of {HBM_TBS} TB/s (bound {bound:.3f} ms)")

    # ---- 2. one prime, 16 continuations ----
    n = 16
    P = min(4096, D - 1)
    tr.drop_engine()
    torch.cuda.empty_cache()
    eng = ca._engine(n)
    assert eng.prefill_capacity >= P, f"prefill capacity {eng.prefill_capacity} < {P}"
    g = torch.Generator(device="cuda").manual_seed(0)
    toks = torch.randint(0, ca.bins, (n, D), device="cuda", generator=g)
    toks[:] = toks[:1]
    yc = torch.randn(n, W, device="cuda", generator=g) * 0.1 if ca.y_cond else None
    xc = torch.zeros(n, 1, W, device="cuda") if ca.x_cond else None
    row = lambda v: None if v is None else v[:1]

    def copies():
        eng.reset(0)
        eng.prefill(n, P, tokens=toks, y_cond=yc, x_cond=xc)

    def one_row():
        eng.reset(0)
        eng.prefill(1, P, tokens=toks, y_cond=row(yc), x_cond=row(xc))
        eng.select([0] * n)
    res = rounds_of({"prefill 16 copies": copies, "prefill 1 + select": one_row}, rounds, 2)
    print(f"one prime of {P} positions, {n} continuations:")
    for k, ts in res.items():
        print(f"  {k:18s}: {fmt(ts)} (min / median of {rounds})")
    print(f"  saved: {min(res['prefill 16 copies']) - min(res['prefill 1 + select']):.1f} ms per window")


if __name__ == "__main__":
    main()
