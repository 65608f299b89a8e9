"""The reference's spectral losses (jukebox/utils/audio_utils.py:8-131) on the fused STFT kernel.

Each STFT config is one `jk_stft_mag_diff` call, which returns per clip the two sums the losses are made of:
sum (|STFT x_in| - |STFT x_out|)^2 and sum |STFT x_in|^2.  The spectrograms themselves are never materialised.
`calculate_bandwidth`, `log_magnitude_loss` and the audio file I/O are not built: evaluation does not call them, and
`hps.bandwidth` is supplied by the caller."""
import torch as t

from .._lib import lib, check, ptr, stream_ptr


class STFTValues:
    """one STFT config: n_fft, hop_length, window_size (win_length), with the sample rate of hps"""
    def __init__(self, hps, n_fft, hop_length, window_size):
        self.sr, self.n_fft, self.hop_length, self.window_size = hps.sr, n_fft, hop_length, window_size


class DefaultSTFTValues(STFTValues):
    """the config of spectral_loss and spectral_convergence: n_fft 2048, hop 256, window 6 hops"""
    def __init__(self, hps):
        super().__init__(hps, 2048, 256, 6 * 256)


def audio_postprocess(x, hps):
    return x


def squeeze(x):
    """[N, T, C] with C in (1, 2) -> mono [N, T] (mean over channels); [N, T] unchanged"""
    if x.dim() == 3:
        assert x.shape[-1] in (1, 2), f"expected 1 or 2 channels, got {x.shape[-1]}"
        x = x.mean(-1)
    if x.dim() != 2:
        raise ValueError(f'Unknown input shape {x.shape}')
    return x


def stft_stats(x_in, x_out, hps):
    """(residual_norm, gt_norm), fp32 [N]: the norms over frames and bins of |STFT x_in| - |STFT x_out| and of
    |STFT x_in| for one STFT config (n_fft, hop_length, window_size), as audio_utils.py:112-131 forms them."""
    a = squeeze(x_in.float()).contiguous()
    b = squeeze(x_out.float()).contiguous()
    if a.shape != b.shape:
        raise ValueError(f"x_in {tuple(a.shape)} and x_out {tuple(b.shape)} differ")
    n, T = a.shape
    window = t.hann_window(hps.window_size, device=a.device)
    resid = t.empty(n, dtype=t.float64, device=a.device)
    norm_a = t.empty(n, dtype=t.float64, device=a.device)
    ws = lib().jk_stft_workspace_bytes(n, T, hps.n_fft, hps.hop_length)
    work = t.empty(max(ws, 8), dtype=t.uint8, device=a.device)
    check(lib().jk_stft_mag_diff(ptr(a), ptr(b), ptr(window), ptr(resid), ptr(norm_a), n, T, hps.n_fft,
                                 hps.hop_length, hps.window_size, ptr(work), work.numel(), stream_ptr()))
    return resid.sqrt().float(), norm_a.sqrt().float()


def convergence(residual_norm, gt_norm, epsilon=2e-3):
    """spectral_convergence (audio_utils.py:124-131) from the two norms of the default config"""
    mask = (gt_norm > epsilon).float()
    return (residual_norm * mask) / t.clamp(gt_norm, min=epsilon)


def spectral_loss(x_in, x_out, hps):
    return stft_stats(x_in, x_out, DefaultSTFTValues(hps))[0]


def multispectral_loss(x_in, x_out, hps):
    """mean over the hps.multispec_loss_* configs of the per-clip spectral residual norm"""
    cfgs = list(zip(hps.multispec_loss_n_fft, hps.multispec_loss_hop_length, hps.multispec_loss_window_size))
    assert len(cfgs) == len(hps.multispec_loss_n_fft) == len(hps.multispec_loss_hop_length) \
        == len(hps.multispec_loss_window_size), "multispec_loss_* lengths differ"
    return sum(stft_stats(x_in, x_out, STFTValues(hps, *c))[0] for c in cfgs) / len(cfgs)


def spectral_convergence(x_in, x_out, hps, epsilon=2e-3):
    return convergence(*stft_stats(x_in, x_out, DefaultSTFTValues(hps)), epsilon=epsilon)
