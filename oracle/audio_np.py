"""fp64 numpy restatement of the reference's STFT losses (jukebox/utils/audio_utils.py:80-131).

torch.stft semantics: center=True with reflect padding of n_fft // 2, 1 + T // hop frames, the periodic Hann window of
win_length zero-padded to n_fft with (n_fft - win_length) // 2 zeros on the left, onesided spectrum (np.fft.rfft)."""
import numpy as np

DEFAULT = (2048, 256, 1536)           # DefaultSTFTValues


def hann(win_length):
    """torch.hann_window (periodic); like torch, a window of length 1 is [1]"""
    if win_length == 1:
        return np.ones(1)
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(win_length) / win_length)


def spec(x, n_fft, hop, win_length):
    """|STFT| of mono signals x [N, T] -> [N, frames, n_fft // 2 + 1] float64"""
    x = np.asarray(x, np.float64)
    T = x.shape[-1]
    assert T > n_fft // 2, "reflect padding needs T > n_fft // 2"
    w = np.zeros(n_fft)
    left = (n_fft - win_length) // 2
    w[left:left + win_length] = hann(win_length)
    xp = np.pad(x, [(0, 0), (n_fft // 2, n_fft // 2)], mode="reflect")
    frames = np.lib.stride_tricks.sliding_window_view(xp, n_fft, axis=-1)[:, ::hop][:, :1 + T // hop]
    return np.abs(np.fft.rfft(frames * w, axis=-1))


def stft_sums(a, b, n_fft, hop, win_length):
    """(resid, norm_a) per clip: sum (|STFT a| - |STFT b|)^2 and sum |STFT a|^2, what jk_stft_mag_diff returns"""
    sa, sb = spec(a, n_fft, hop, win_length), spec(b, n_fft, hop, win_length)
    return ((sa - sb) ** 2).sum(axis=(1, 2)), (sa ** 2).sum(axis=(1, 2))


def squeeze(x):
    x = np.asarray(x, np.float64)
    return x.mean(-1) if x.ndim == 3 else x


def spectral_loss(x_in, x_out, cfg=DEFAULT):
    return np.sqrt(stft_sums(squeeze(x_in), squeeze(x_out), *cfg)[0])


def multispectral_loss(x_in, x_out, n_ffts, hops, windows):
    losses = [spectral_loss(x_in, x_out, cfg) for cfg in zip(n_ffts, hops, windows)]
    return sum(losses) / len(losses)


def spectral_convergence(x_in, x_out, epsilon=2e-3):
    resid, norm_a = stft_sums(squeeze(x_in), squeeze(x_out), *DEFAULT)
    gt, res = np.sqrt(norm_a), np.sqrt(resid)
    return res * (gt > epsilon) / np.maximum(gt, epsilon)
