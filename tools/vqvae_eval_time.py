"""Time VQVAE.forward (evaluation: losses and metrics) at C5 geometry, and its spectral losses on the fused STFT kernel
(jk_stft_mag_diff) against the same losses composed from fp32 torch.stft on cuFFT, with CUDA events.

    python tools/vqvae_eval_time.py [--clips 16] [--samples 1048576] [--rounds 3] [--out DIR]

Geometry: the `vqvae` hparams (3 levels) with synthetic weights (bench.synth_fill, random codebooks), `clips` clips of
`samples` samples.  Kernel comparison: one spectral_loss + multispectral_loss pass of one level (the four STFT configs)
on both routes, on the same signals (x and its level-0 reconstruction); the routes alternate for `rounds` rounds after a
warm-up of both, and the min / median / max are printed with the maximum relative difference of the per-clip losses.
The kernel's bound: 5 n log2 n FLOP per complex FFT of n points, one FFT per frame (the two signals share it), against
the 67 TFLOP/s FP32 figure of the H100 SXM data sheet.  Whole forward: VQVAE.forward end to end, then its four phases
(encoders, bottleneck, decoders, losses) timed one by one.  Prints the GPU's name and power limit in the same run.
"""
import argparse
import contextlib
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import synth_fill  # noqa: E402

FP32_PEAK = 67e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def stats(v):
    return dict(ms_min=round(min(v), 3), ms_median=round(statistics.median(v), 3), ms_max=round(max(v), 3))


def configs(hps):
    return [(2048, 256, 1536)] + list(zip(hps.multispec_loss_n_fft, hps.multispec_loss_hop_length,
                                          hps.multispec_loss_window_size))


def kernel_route(x, y, hps):
    """per clip [spectral_loss, multispectral_loss] of audio_utils on jk_stft_mag_diff"""
    from jukebox_b200.utils.audio_utils import spectral_loss, multispectral_loss
    return torch.stack([spectral_loss(x, y, hps), multispectral_loss(x, y, hps)])


def torch_route(x, y, hps):
    """the same two losses from fp32 torch.stft magnitudes (cuFFT), the way the reference composes them"""
    a, b = x.float().mean(-1), y.float().mean(-1)
    out = []
    for n_fft, hop, win in configs(hps):
        w = torch.hann_window(win, device=x.device)
        sa = torch.stft(a, n_fft, hop, win_length=win, window=w, return_complex=True).abs()
        sb = torch.stft(b, n_fft, hop, win_length=win, window=w, return_complex=True).abs()
        out.append((sa - sb).reshape(a.shape[0], -1).pow(2).sum(-1).sqrt())
    return torch.stack([out[0], sum(out[1:]) / len(out[1:])])


def fft_flop(clips, samples, hps):
    return sum(clips * (1 + samples // hop) * 5 * n * math.log2(n) for n, hop, _ in configs(hps))


def main():
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae
    from jukebox_b200.vqvae import vqvae as vqvae_mod
    from jukebox_b200.utils import audio_utils
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--samples", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vqvae_eval_time.py measures on a CUDA device; none found")
    gpu = gpu_info()
    print(f"GPU: {gpu}", flush=True)
    hps = setup_hparams("vqvae", dict(sample_length=a.samples, restore_vqvae=""))
    with contextlib.redirect_stdout(sys.stderr), torch.device("cuda"):
        vq = make_vqvae(hps, "cuda")
    synth_fill(vq, 5)
    g = torch.Generator(device="cuda").manual_seed(1)
    with torch.no_grad():
        for blk in vq.bottleneck.level_blocks:
            blk.k.copy_(torch.randn(blk.k.shape, device="cuda", generator=g))
    vq.eval()
    x = (2 * torch.rand(a.clips, a.samples, 1, device="cuda", generator=g) - 1) * 0.5
    hps.bandwidth = dict(l1=0.25, l2=1 / 12 * 0.25, spec=1000.0)

    with torch.no_grad():
        x_out, _, _ = vq(x, hps, loss_fn=hps.loss_fn)         # warm-up of the whole forward, every shape
        kernel_route(x, x_out, hps)
        torch_route(x, x_out, hps)
        ms = {"kernel": [], "torch": []}
        outs = {}
        for _ in range(a.rounds):
            for name, fn in (("kernel", kernel_route), ("torch", torch_route)):
                t, outs[name] = timed(lambda: fn(x, x_out, hps))
                ms[name].append(t)
        diff = float(((outs["kernel"].double() - outs["torch"].double()).abs() / outs["torch"].double().abs()).max())
        flop = fft_flop(a.clips, a.samples, hps)
        kmed = statistics.median(ms["kernel"])
        r = dict(gpu=gpu, clips=a.clips, samples=a.samples, configs=configs(hps),
                 kernel=dict(**stats(ms["kernel"]), tflops=round(flop / (kmed * 1e-3) / 1e12, 2),
                             fp32_bound_ms=round(flop / FP32_PEAK * 1e3, 3),
                             share_of_fp32_peak=round(flop / FP32_PEAK * 1e3 / kmed, 3)),
                 torch_stft=stats(ms["torch"]), speedup=round(statistics.median(ms["torch"]) / kmed, 2),
                 max_rel_diff_routes=diff, fft_gflop_per_level=round(flop / 1e9, 2))
        print(json.dumps(dict(spectral_pass_one_level=r)), flush=True)

        phases = {k: [] for k in ("forward", "encoders", "bottleneck", "decoders", "losses")}
        for _ in range(a.rounds):
            t, _ = timed(lambda: vq(x, hps, loss_fn=hps.loss_fn))
            phases["forward"].append(t)
            x_in = vq.preprocess(x)
            t, xs = timed(lambda: [vq.encoders[l](x_in)[-1] for l in range(vq.levels)])
            phases["encoders"].append(t)
            t, (_, xq, _, _) = timed(lambda: vq.bottleneck(xs))
            phases["bottleneck"].append(t)
            t, x_outs = timed(lambda: [vq.decoders[l](xq[l:l + 1], all_levels=False) for l in range(vq.levels)])
            phases["decoders"].append(t)

            def losses():
                for l in range(vq.levels):
                    vqvae_mod._loss_fn(hps.loss_fn, x, x_outs[l], hps)
                    audio_utils.stft_stats(x, x_outs[l], audio_utils.DefaultSTFTValues(hps))
                    audio_utils.multispectral_loss(x, x_outs[l], hps)
                for name in ("l2", "l1", "linf"):
                    vqvae_mod._loss_fn(name, x, x_outs[0], hps)
            t, _ = timed(losses)
            phases["losses"].append(t)
            del xs, xq, x_outs
        f = dict(gpu=gpu, clips=a.clips, samples=a.samples, levels=vq.levels, loss_fn=hps.loss_fn,
                 **{k: stats(v) for k, v in phases.items()})
        print(json.dumps(dict(vqvae_forward=f)), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "vqvae_eval_time.json"), "w") as fh:
            json.dump(dict(spectral_pass_one_level=r, vqvae_forward=f), fh, indent=1)


if __name__ == "__main__":
    main()
