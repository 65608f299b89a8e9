"""CPU checks of the VQVAE.forward fixture (tests/golden/vqvae_forward_3level.npz, written by
oracle/make_golden_vqvae_forward.py from the live reference): the fp64 numpy STFT losses of oracle/audio_np.py reproduce
every spectral metric the reference's fp32 torch.stft gave, which pins the padding, the window centring and the frame
count the GPU kernel is tested against.  Also: the host's argument checks that need no GPU."""
import numpy as np
import pytest
import torch

from golden_util import Fixture
from oracle import audio_np


def _spectral_metrics(fx, nonrel):
    c = fx.cfg
    bw = c["bandwidth"]
    x = fx["x"]
    out, spec_sum, multi_sum = {}, 0.0, 0.0
    for level in reversed(range(c["levels"])):
        x_out = fx[f"x_out_l{level + 1}"]
        if nonrel:
            spec = np.mean(audio_np.spectral_loss(x, x_out) / bw["spec"])
        else:
            spec = np.mean(audio_np.spectral_convergence(x, x_out))
        multi = np.mean(audio_np.multispectral_loss(x, x_out, c["multispec_loss_n_fft"], c["multispec_loss_hop_length"],
                                                    c["multispec_loss_window_size"]) / bw["spec"])
        out[f"spectral_loss_l{level + 1}"] = spec
        out[f"multispectral_loss_l{level + 1}"] = multi
        spec_sum += spec
        multi_sum += multi
    out["spectral_loss"] = spec_sum
    out["multispectral_loss"] = multi_sum
    out["spectral_convergence"] = np.mean(audio_np.spectral_convergence(x, fx["x_out_l1"]))
    return out


def test_numpy_oracle_reproduces_reference_spectral_metrics():
    fx = Fixture("vqvae_forward_3level")
    assert len(fx.cfg["cases"]) == 8
    for case in fx.cfg["cases"]:
        assert len(case["keys"]) == 17
        want = _spectral_metrics(fx, case["use_nonrelative_specloss"])
        for k, v in want.items():
            ref = float(fx[f"{case['case']}/{k}"])
            assert abs(v - ref) <= 1e-5 * abs(ref), (case["case"], k, v, ref)


def test_oracle_frame_count_and_window_centring():
    """torch.stft on CPU (fp64) against the oracle for an odd window and a T that is not a multiple of hop"""
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 1001))
    for n_fft, hop, win in [(256, 50, 101), (512, 120, 512), (256, 7, 1)]:
        ref = torch.stft(torch.from_numpy(x), n_fft, hop, win_length=win, window=torch.hann_window(win, dtype=torch.float64),
                         return_complex=True).abs().numpy().transpose(0, 2, 1)
        got = audio_np.spec(x, n_fft, hop, win)
        assert got.shape == ref.shape == (2, 1 + 1001 // hop, n_fft // 2 + 1)
        np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-9)


def test_stft_workspace_bytes_rejects_bad_sizes():
    from jukebox_b200._lib import lib
    assert lib().jk_stft_workspace_bytes(16, 1 << 20, 512, 50) > 0
    assert lib().jk_stft_workspace_bytes(16, 1 << 20, 1000, 50) == 0
    assert lib().jk_stft_workspace_bytes(16, 1 << 20, 8192, 50) == 0
    assert lib().jk_stft_workspace_bytes(16, 1 << 20, 512, 0) == 0
    # the frame-to-CTA split depends on the clip length and config only: the workspace is linear in the batch
    one = lib().jk_stft_workspace_bytes(1, 1 << 20, 512, 50)
    assert lib().jk_stft_workspace_bytes(16, 1 << 20, 512, 50) == 16 * one


def test_forward_requires_eval_mode_and_bandwidth():
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae
    from jukebox_b200.vqvae.bottleneck import BottleneckBlock
    hps = setup_hparams("vqvae", dict(restore_vqvae="", sample_length=128 * 40))
    vq = make_vqvae(hps, "cpu")
    x = torch.zeros(1, 128 * 40, 1)
    with pytest.raises(NotImplementedError):
        vq.train()(x, hps)
    with pytest.raises(ValueError, match="bandwidth"):
        vq.eval()(x, hps)
    with pytest.raises(NotImplementedError):
        BottleneckBlock(16, 64, 0.99)(torch.zeros(1, 4, 64), update_k=True)
