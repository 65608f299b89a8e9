"""Generate tests/golden/vqvae_forward_3level.npz: the live reference's VQVAE.forward (jukebox/vqvae/vqvae.py:150-228)
in eval mode, on CPU, for every loss_fn and both settings of use_nonrelative_specloss.

    python -m oracle.make_golden_vqvae_forward

One shim is local to this script: current torch rejects the reference's `t.stft(...)` without `return_complex`, so
torch.stft is wrapped to return view_as_real(stft(..., return_complex=True)), the real / imag pairs the reference's
torch returned.  Stored: the config, x, the per-level reconstructions x_out_l1..3 (x_out is x_out_l1), and per case
every metric and the loss.  The weights are the synthetic ones of oracle/synth.py (name, shape, seed)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.make_golden import load_synth, save   # noqa: E402  (imports the CPU-shimmed reference)
from oracle import audio_np                        # noqa: E402
import torch as t                                  # noqa: E402

_stft = t.stft


def _stft_real(*args, **kwargs):
    kwargs["return_complex"] = True
    return t.view_as_real(_stft(*args, **kwargs))


LOSS_FNS = ("lmix", "l1", "l2", "linf")


def main(seed=3, bs=2, sample_length=128 * 40):
    from jukebox.hparams import setup_hparams
    from jukebox.make_models import make_vqvae
    t.stft = _stft_real
    overrides = dict(sample_length=sample_length)
    hps = setup_hparams("vqvae", dict(restore_vqvae="", **overrides))
    vq = make_vqvae(hps, "cpu")
    named = load_synth(vq, seed)
    vq.eval()
    g = t.Generator().manual_seed(seed)
    x = 2 * t.rand(bs, hps.sample_length, 1, generator=g) - 1
    xn = x.numpy()[..., 0].astype(np.float64)
    # the dataset statistics train.py:calculate_bandwidth would give, taken from x itself
    hps.bandwidth = dict(l1=float(np.abs(xn).mean()), l2=float(xn.var()),
                         spec=float(np.sqrt((audio_np.spec(xn, *audio_np.DEFAULT) ** 2).sum(axis=(1, 2))).mean()))
    arrays = dict(x=x)
    with t.no_grad():
        x_in = vq.preprocess(x)
        xs = [vq.encoders[level](x_in)[-1] for level in range(vq.levels)]
        _, xs_quantised, _, _ = vq.bottleneck(xs)
        for level in range(vq.levels):
            arrays[f"x_out_l{level + 1}"] = vq.postprocess(vq.decoders[level](xs_quantised[level:level + 1],
                                                                              all_levels=False))
    cases = []
    for loss_fn in LOSS_FNS:
        for nonrel in (True, False):
            case = f"{loss_fn}_{'nonrel' if nonrel else 'conv'}"
            hps.use_nonrelative_specloss = nonrel
            with t.no_grad():
                x_out, loss, metrics = vq(x, hps, loss_fn=loss_fn)
            assert t.equal(x_out, arrays["x_out_l1"]), case
            arrays[f"{case}/loss"] = loss
            for k, v in metrics.items():
                arrays[f"{case}/{k}"] = v
            cases.append(dict(case=case, loss_fn=loss_fn, use_nonrelative_specloss=nonrel, keys=sorted(metrics)))
            print(case, f"loss {float(loss):.6g}", len(metrics), "metrics")
    arrays["x_out"] = arrays["x_out_l1"]
    cfg = dict(hps_name="vqvae", overrides=overrides, seed=seed, levels=hps.levels, bandwidth=hps.bandwidth,
               cases=cases, linf_k=hps.linf_k, lmix_l1=hps.lmix_l1, lmix_l2=hps.lmix_l2, lmix_linf=hps.lmix_linf,
               multispec_loss_n_fft=list(hps.multispec_loss_n_fft),
               multispec_loss_hop_length=list(hps.multispec_loss_hop_length),
               multispec_loss_window_size=list(hps.multispec_loss_window_size))
    save("vqvae_forward_3level", cfg, named, **arrays)


if __name__ == "__main__":
    main()
