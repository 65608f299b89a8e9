"""Time one window of lyric alignment (jukebox_b200.align.hop_weights: what get_alignment runs per top-level window) on the
fp16 route (attention recorded by the fp16 prefill) and on the fp32 route (the fp32 forward-mode path), with CUDA events.

    python tools/align_time.py [--items 16] [--out DIR]

Geometry: the top-level priors of 1b_lyrics and 5b_lyrics at their full width, heads, context and lyric length, with
synthetic weights (bench.synth_fill, the scale rules of oracle/synth.py).  The stacks are cut to the first layers that
contain a layer of the alignment layer's kind (1b_lyrics: 16 layers, layer 15 is a prime layer like layer 63; 5b_lyrics:
19 layers, layer 18 is an encoder-decoder layer like layer 68), so that the fp32 route fits a short run; the time per
layer is reported beside the window time.  The fp16 route runs the window's items in one z_forward call (as many as
one prefill takes), the fp32 route item by item, as get_alignment does.  Prints one JSON line per (model, route) and
the GPU's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import WORKLOADS, hps_pair, make_labels, synth_fill  # noqa: E402
from jukebox_b200 import align  # noqa: E402

MODELS = {
    # workload: (layers kept, recorded layer, the full model's depth)
    "1b_lyrics": (16, 15, 72),
    "5b_lyrics": (19, 18, 79),
}


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def build(wl, depth, seed=0):
    from jukebox_b200.make_models import make_vqvae, make_prior
    w = dict(WORKLOADS[wl])
    w["prior"] = (w["prior"][0], dict(w["prior"][1], prior_depth=depth))
    vq_h, pr_h = hps_pair(w)
    with torch.device("cuda"):
        prior = make_prior(pr_h, make_vqvae(vq_h, "cuda"), "cuda")
    synth_fill(prior, seed)
    return prior, pr_h


def time_window(prior, z, y, fp16):
    # warm-up: the engines are built for the batch the timed call runs (fp16: every item in one prefill call), the fp32
    # path is built, kernels are loaded.  The fp32 route runs item by item, so one item warms it up.
    warm = z.shape[0] if fp16 else 1
    align.hop_weights(prior, z[:warm], y[:warm], fp16)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    w = align.hop_weights(prior, z, y, fp16)               # ends in a device -> host copy
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3, w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=16)
    ap.add_argument("--models", default=",".join(MODELS))
    ap.add_argument("--out", default=None, help="directory for the JSON results")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("align_time.py measures on a CUDA device; none found")
    gpu = gpu_info()
    print(f"GPU: {gpu}", flush=True)
    results = []
    for wl in a.models.split(","):
        depth, layer, full_depth = MODELS[wl]
        prior, hps = build(wl, depth)
        tr = prior.prior.transformer
        assert tr._attn_mods[layer].attn_func in (6, 7)
        prior.alignment_layer, prior.alignment_head = layer, 0
        g = torch.Generator().manual_seed(1)
        z = torch.randint(0, prior.l_bins, (a.items, prior.n_ctx), generator=g).cuda()
        y = make_labels(prior, hps, a.items, 1).cuda()
        times = {}
        for fp16 in (True, False):
            s, w = time_window(prior, z, y, fp16)
            times[fp16] = (s, w)
            eng_batch = tr._engine.max_batch if tr._engine is not None else 0     # samples the decoder's engine took
            for m in (prior.prior, getattr(prior, "prime_prior", None)):     # decoder and lyric encoder (5b_lyrics)
                if m is not None:
                    m.transformer.drop_engine()                # free the route's engines / fp32 state before the next
            torch.cuda.empty_cache()
            per_call = (prior.prior.items_per_prefill(a.items) or 1) if fp16 else 1
            r = dict(model=wl, route="fp16" if fp16 else "fp32", items=a.items, items_per_call=per_call,
                     engine_batch=eng_batch, n_ctx=prior.n_ctx, layers=depth,
                     recorded_layer=layer, attn_func=tr._attn_mods[layer].attn_func, window_s=round(s, 4),
                     per_layer_ms=round(1e3 * s / depth, 2), gpu=gpu)
            print(json.dumps(r), flush=True)
            results.append(r)
        d = float(abs(times[True][1] - times[False][1]).max())
        print(f"{wl}: fp32 / fp16 window time {times[False][0] / times[True][0]:.1f}x; max|w16 - w32| {d:.2e}", flush=True)
        del prior, tr
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "align_time.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
