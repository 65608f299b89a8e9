"""Cost of scoring tokens at 1b_lyrics geometry (synthetic weights), with the card it ran on.

1. The x_out head of SimplePrior.score over a full window (16 and 32 items x 8576 positions): the fused route
   (jk_xout_logprob: split-precision wgmma product + log-softmax at the target, no logits tensor) against the composed
   one (f32.linear_nk -> [M, bins] fp32 logits -> torch.log_softmax -> gather), on the same activations, alternated.
   Useful TFLOP/s counts 2 M W bins (the fused kernel issues three fp16 MMAs per useful one).  Then one whole
   SimplePrior.score call at 16 items (activations + head).
2. What get_logprobs=True adds per decode position at 500 / 4000 / 8000: one decode step + the sampling launch, with
   the unscored and the scored draw, alternated.  The decode step itself is the same call either way.

    python tools/score_time.py [--small]
"""
import contextlib
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

FP16_TFLOPS = 989.0     # H100 SXM data sheet, dense FP16 tensor
FP32_TFLOPS = 67.0


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    assert torch.cuda.is_available(), "score_time needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(f"card: {torch.cuda.get_device_name()} | nvidia-smi: {q.stdout.strip().splitlines()[0] if q.stdout else 'n/a'}")
    small = "--small" in sys.argv
    wl = bench.SMALL if small else bench.WORKLOADS["1b_lyrics"]
    with contextlib.redirect_stdout(sys.stderr):
        prior, hps = bench.build_prior(wl)
    from jukebox_b200.score import xout_logprob
    from jukebox_b200.transformer import f32
    from jukebox_b200.transformer.ops import sample_categorical, sample_categorical_scored
    ca = prior.prior
    D, W, bins = ca.input_dims, ca.width, ca.bins
    w = ca.x_out.weight
    g = torch.Generator(device="cuda").manual_seed(0)

    # ---- 1. the head over a full window ----
    for n in (16, 32):
        M = n * D
        h = torch.randn(M, W, device="cuda", generator=g)
        tg = torch.randint(0, bins, (M,), device="cuda", generator=g)
        fused = lambda: xout_logprob(h, w, tg)
        composed = lambda: torch.log_softmax(f32.linear_nk(h, w), -1).gather(1, tg[:, None])[:, 0]
        a, b = fused(), composed()
        d = (a - b).abs()
        top = torch.topk(d, 16).indices          # where the routes differ most: which one is off, against fp64
        ref = torch.log_softmax(h[top].double() @ w.double().T, -1).gather(1, tg[top][:, None])[:, 0]
        ea, eb = float((a[top].double() - ref).abs().max()), float((b[top].double() - ref).abs().max())
        d = float(d.max())
        del a, b
        ts = {"fused": [], "composed": []}
        for _ in range(3):
            ts["fused"].append(timed(fused, 3))
            ts["composed"].append(timed(composed, 3))
        flop = 2.0 * M * W * bins
        for k, v in ts.items():
            ms = min(v)
            print(f"head n={n} M={M} W={W} bins={bins} {k:8s}: {ms:8.2f} ms (min of {['%.2f' % x for x in v]}) "
                  f"useful {flop / ms / 1e9:6.1f} TFLOP/s = {flop / ms / 1e9 / FP16_TFLOPS * 100:4.1f} % of FP16 "
                  f"{FP16_TFLOPS:.0f}" + (f", {3 * flop / ms / 1e9:6.1f} TFLOP/s of fp16 MMA issued" if k == "fused" else
                                          f", {flop / ms / 1e9 / FP32_TFLOPS * 100:4.1f} % of FP32 {FP32_TFLOPS:.0f}"))
        print(f"head n={n}: speed-up {min(ts['composed']) / min(ts['fused']):.1f}x, max |dlogp| between routes {d:.1e}; "
              f"on the 16 rows where they differ most, |dlogp| vs fp64: fused {ea:.1e}, composed {eb:.1e}")
        del h, tg
        torch.cuda.empty_cache()

    # whole SimplePrior.score (activations + head) at 16 items
    n = 16
    y = bench.make_labels(prior, hps, n, 0)
    y = None if y is None else y.cuda()
    z = torch.randint(0, prior.l_bins, (n, prior.n_ctx), device="cuda", generator=g)
    cap = ca.transformer.prefill_capacity(n)
    how = "prefill" if D <= cap else "stepped (beyond the prefill capacity)"
    prior.score(z, [], y)
    torch.cuda.synchronize()
    ms = timed(lambda: prior.score(z, [], y), 1)
    print(f"SimplePrior.score n={n} x {D} positions ({how}, capacity {cap}): {ms:.1f} ms")

    # ---- 2. get_logprobs per decode position ----
    eng = ca._engine(n)
    toks = torch.randint(0, bins, (n, D), device="cuda", generator=g)
    lbuf = torch.empty(n, bins, device="cuda")
    lp = torch.zeros(n, D, device="cuda")
    yc = torch.randn(n, W, device="cuda", generator=g) if ca.y_cond else None
    xc = torch.zeros(n, 1, W, device="cuda") if ca.x_cond else None
    lb = f32.linear_nk(xc.reshape(n, W), w).view(n, 1, bins) if xc is not None and eng.has_logits_gemm else None
    if ca.transformer.encoder_dims:
        eng.set_encoder_kv(torch.randn(n, ca.transformer.encoder_dims, W, device="cuda"))
    for pos0 in (500, 4000, 8000):
        pos0 = min(pos0, D - 200)
        res = {"off": [], "on": []}
        for rnd in range(3):
            for k in ("off", "on"):
                eng.reset(pos0)

                def one():
                    p = eng.position
                    eng.step(n, tokens=toks, y_cond=yc, x_cond=xc, logits=lbuf, logit_bias=lb)
                    if k == "on":
                        sample_categorical_scored(lbuf, lbuf, 0.99, 1234, p, toks, lp)
                    else:
                        sample_categorical(lbuf, 0.99, 1234, p, toks)
                for _ in range(5):
                    one()
                res[k].append(timed(one, 25) * 1000)
        off, on = min(res["off"]), min(res["on"])
        print(f"decode position {pos0}: step + draw {off:.1f} us, step + scored draw {on:.1f} us, "
              f"get_logprobs adds {on - off:+.1f} us ({(on - off) / off * 100:+.2f} %) "
              f"[off {['%.1f' % x for x in res['off']]}, on {['%.1f' % x for x in res['on']]}]")


if __name__ == "__main__":
    main()
