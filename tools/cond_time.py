"""Time the upsampler Conditioner (SimplePrior.get_cond: the x_cond of one window) on the wide tensor-core convs
(jk_conv1d_tc_wide) and on the exact-FMA route (use_tensor_cores(..., False)), with CUDA events.

    python tools/cond_time.py [--priors upsampler_level_0,upsampler_level_1,small_upsampler] [--batches 16,32]
                              [--rounds 3] [--out DIR]

Geometry: the priors' own hparams and window (n_ctx 8192) with synthetic weights (bench.synth_fill); the transformer is
cut to one layer, since only the conditioning runs.  After a warm-up of both routes at every batch size, the two routes
alternate in one process for `rounds` rounds; the min / median / max per window are printed with the useful TFLOP/s
(2 FLOP per MAC of the convs, counted from their shapes; the split-precision kernel issues 3 fp16 products per MAC,
reported separately as the tensor-core rate) and the max relative difference between the routes' x_cond
(max|a - b| / max|b|).  Prints the GPU's name and power limit in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import hps_pair, make_labels, synth_fill  # noqa: E402

PRIORS = {
    # prior: (vq-vae hparams, sample length of one 8192-token window at the prior's level, prior overrides)
    "upsampler_level_0": ("vqvae", 8192 * 8, dict(prior_depth=1)),
    "upsampler_level_1": ("vqvae", 8192 * 32, dict(prior_depth=1)),
    "small_upsampler": ("small_vqvae", 8192 * 32, dict(labels=False, level=0, levels=2, prior_depth=1)),
}


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def build(name, seed=0):
    from jukebox_b200.make_models import make_vqvae, make_prior
    vq, length, over = PRIORS[name]
    vq_h, pr_h = hps_pair(dict(vq=(vq, dict(sample_length=length)), prior=(name, over)))
    with torch.device("cuda"):
        prior = make_prior(pr_h, make_vqvae(vq_h, "cuda"), "cuda")
    synth_fill(prior, seed)
    return prior.eval(), pr_h


def count_macs(cond, run):
    """multiply-accumulates of the Conditioner's convs in one call of `run`, from the shapes they see"""
    from jukebox_b200.vqvae.ops_cl import Conv1d, ConvTranspose1d
    total = [0]

    def hook(m, args, out):
        x = args[0]
        n, t_in, c_in = x.shape
        if isinstance(m, ConvTranspose1d):
            total[0] += n * (2 * t_in) * 2 * c_in * m.n_out        # every output position takes 2 of the 4 taps
        else:
            total[0] += n * (t_in // m.stride) * m.k * c_in * m.n_out

    hs = [m.register_forward_hook(hook) for m in cond.modules() if isinstance(m, (Conv1d, ConvTranspose1d))]
    run()
    for h in hs:
        h.remove()
    return total[0]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    from jukebox_b200.vqvae.resnet import use_tensor_cores
    ap = argparse.ArgumentParser()
    ap.add_argument("--priors", default=",".join(PRIORS))
    ap.add_argument("--batches", default="16,32")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON results")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cond_time.py measures on a CUDA device; none found")
    gpu = gpu_info()
    print(f"GPU: {gpu}", flush=True)
    results = []
    for name in a.priors.split(","):
        prior, hps = build(name)
        cond = prior.conditioner_blocks[0]
        up = prior.cond_level
        batches = [int(b) for b in a.batches.split(",")]
        inputs = {}
        for n in batches:
            g = torch.Generator().manual_seed(n)
            zc = [torch.randint(0, prior.l_bins, (n, *prior.z_shapes[up]), generator=g).cuda()]
            y = make_labels(prior, hps, n, 1).cuda() if prior.y_cond else None
            inputs[n] = (zc, y)
        with torch.no_grad():
            for n in batches:                                   # warm-up: both routes, every shape
                for on in (True, False):
                    use_tensor_cores(cond, on)
                    prior.get_cond(*inputs[n])
            for n in batches:
                run = lambda: prior.get_cond(*inputs[n])[0]     # noqa: E731
                macs = count_macs(cond, run)
                ms = {True: [], False: []}
                outs = {}
                for _ in range(a.rounds):
                    for on in (True, False):
                        use_tensor_cores(cond, on)
                        t, outs[on] = timed(run)
                        ms[on].append(t)
                diff = float((outs[True].double() - outs[False].double()).abs().max() / outs[False].double().abs().max())
                r = dict(prior=name, samples=n, positions=int(outs[True].shape[1]), width=int(outs[True].shape[2]),
                         macs=macs, rel_diff_routes=diff, gpu=gpu)
                for on, tag in ((True, "tensor_cores"), (False, "exact")):
                    v = ms[on]
                    med = statistics.median(v)
                    r[tag] = dict(ms_min=round(min(v), 2), ms_median=round(med, 2), ms_max=round(max(v), 2),
                                  useful_tflops=round(2 * macs / (med * 1e-3) / 1e12, 1))
                r["tensor_cores"]["split_product_tflops"] = round(3 * r["tensor_cores"]["useful_tflops"], 1)
                r["speedup"] = round(statistics.median(ms[False]) / statistics.median(ms[True]), 2)
                print(json.dumps(r), flush=True)
                results.append(r)
        use_tensor_cores(cond, True)
        del prior, cond, inputs
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "cond_time.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
