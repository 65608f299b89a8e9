"""Cost of guided sampling at 1b_lyrics geometry (synthetic weights), with the card it ran on.

Per drawn position (one engine step with logits + the draw), the engine standing at t in {500, 4000, 8000}:
  guided 16   - 16 guided items: one step of 32 rows + one jk_sample_guided launch of 16 pairs;
  plain 16    - 16 unguided items: one step of 16 rows (an engine of 16 rows) + jk_sample_categorical;
  plain 32    - 32 unguided items: one step of 32 rows + jk_sample_categorical.
The x_cond logit bias is passed as SamplingWindow passes it.  K consecutive positions are timed per round and divided
by K.  Then the draw alone, 16 pairs of 2127 bins: the fused launch against the composed route (torch g = c + s (c - u),
jk_filter_logits when a filter is set, jk_sample_categorical, a copy of the token column to the alternative rows).
The routes alternate within every round; every shape runs before the timed rounds; CUDA events; min / median.

    python tools/guide_time.py [--small] [--rounds R]
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


def fmt(ts, per=1, unit="us"):
    return f"{min(ts) * 1e3 / per:9.1f} / {statistics.median(ts) * 1e3 / per:9.1f} {unit}"


def main():
    from jukebox_b200.transformer import f32
    from jukebox_b200.transformer.ops import filter_logits_scaled, sample_categorical, sample_guided
    assert torch.cuda.is_available(), "guide_time needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(f"card: {torch.cuda.get_device_name()} | nvidia-smi: {q.stdout.strip().splitlines()[0] if q.stdout else 'n/a'}")
    small = "--small" in sys.argv
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 5
    wl = bench.SMALL if small else bench.WORKLOADS["1b_lyrics"]
    with contextlib.redirect_stdout(sys.stderr):
        prior, _ = bench.build_prior(wl)
    ca = prior.prior
    D, W, B = ca.input_dims, ca.width, ca.bins
    eng16 = ca._engine(16)
    ca.transformer._engine = None                 # a second engine, of 32 rows, next to the 16-row one
    eng32 = ca._engine(32)
    g = torch.Generator(device="cuda").manual_seed(0)
    toks = torch.randint(0, B, (32, D), device="cuda", generator=g)
    yc = torch.randn(32, W, device="cuda", generator=g) * 0.1 if ca.y_cond else None
    xc = torch.randn(32, D, W, device="cuda", generator=g) * 0.01 if ca.x_cond else None
    bias = None
    if ca.add_cond_after_transformer and xc is not None and eng32.has_logits_gemm:
        bias = f32.linear_nk(xc.reshape(-1, W), ca.x_out.weight).view(32, D, B)
    print(f"1b_lyrics geometry: {ca.depth} layers, width {W}, {D} positions, {B} bins")
    lbuf = torch.empty(32, B, device="cuda")
    K = 16
    rows = lambda v, n: None if v is None else v[:n]

    def run(eng, n, t, draw):
        def fn():
            for k in range(K):
                eng.step(n, tokens=toks, y_cond=rows(yc, n), x_cond=rows(xc, n), logits=lbuf, logit_bias=rows(bias, n))
                draw(t + k)
        return fn

    cases = {
        "guided 16 (32 rows)": (eng32, 32, lambda p: sample_guided(lbuf[:16], lbuf[16:], 2.0, 1.0, 0, 0.0, 7, p,
                                                                   toks[:16], toks[16:])),
        "plain 16": (eng16, 16, lambda p: sample_categorical(lbuf[:16], 1.0, 7, p, toks[:16])),
        "plain 32": (eng32, 32, lambda p: sample_categorical(lbuf, 1.0, 7, p, toks)),
    }
    for t in ((16, 64, 200) if D < 2048 else (500, 4000, 8000)):
        t = min(t, D - K)
        for eng, n, draw in cases.values():      # warm-up of every shape
            eng.reset(t)
            timed(run(eng, n, t, draw))
        res = {k: [] for k in cases}
        for _ in range(rounds):
            for k, (eng, n, draw) in cases.items():
                eng.reset(t)
                res[k].append(timed(run(eng, n, t, draw)))
        print(f"position {t}, per drawn position (min / median of {rounds} rounds of {K} positions):")
        for k, ts in res.items():
            print(f"  {k:20s}: {fmt(ts, K)}")
        print(f"  guided 16 / plain 16: x{min(res['guided 16 (32 rows)']) / min(res['plain 16']):.2f}   "
              f"guided 16 / plain 32: x{min(res['guided 16 (32 rows)']) / min(res['plain 32']):.2f}")

    # the draw alone: 16 pairs, fused against composed
    c = torch.randn(16, B, device="cuda", generator=g) * 3
    u = torch.randn(16, B, device="cuda", generator=g) * 3
    tk = torch.zeros(32, 64, dtype=torch.long, device="cuda")
    fbuf = torch.empty(16, B, device="cuda")
    R = 200
    for name, top_k, top_p in (("no filter", 0, 0.0), ("top-p 0.95", 0, 0.95), ("top-k 64", 64, 0.0)):
        def fused():
            for i in range(R):
                sample_guided(c, u, 2.0, 0.9, top_k, top_p, 7, i % 64, tk[:16], tk[16:])

        def composed():
            for i in range(R):
                gg = c + 2.0 * (c - u)
                if top_k or top_p:
                    sample_categorical(filter_logits_scaled(gg, 0.9, top_k, top_p, fbuf), 1.0, 7, i % 64, tk[:16])
                else:
                    sample_categorical(gg, 0.9, 7, i % 64, tk[:16])
                tk[16:, i % 64] = tk[:16, i % 64]
        routes = {"fused": fused, "composed": composed}
        for fn in routes.values():
            timed(fn)
        res = {k: [] for k in routes}
        for _ in range(rounds):
            for k, fn in routes.items():
                res[k].append(timed(fn))
        print(f"draw of 16 pairs x {B} bins, {name} (min / median per launch of {rounds} rounds of {R}): "
              f"fused {fmt(res['fused'], R)}, composed {fmt(res['composed'], R)}, "
              f"x{min(res['composed']) / min(res['fused']):.2f}")


if __name__ == "__main__":
    main()
