"""GPU: VQVAE.forward against the live reference's outputs (tests/golden/vqvae_forward_3level.npz), and the fused STFT
kernel jk_stft_mag_diff against the fp64 numpy oracle (oracle/audio_np.py): C5 geometry, edge shapes, determinism and
batch independence, rejected input."""
import types

import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err
from oracle import audio_np
from oracle.vqvae_np import quantise

pytestmark = pytest.mark.gpu

CONFIGS = [(2048, 256, 1536), (2048, 240, 1200), (1024, 120, 600), (512, 50, 240)]   # default + multispec


def _sums(a, b, n_fft, hop, win):
    """jk_stft_mag_diff on [n, T] CUDA signals -> (resid, norm_a) float64 numpy"""
    from jukebox_b200._lib import lib, check, ptr, stream_ptr
    n, T = a.shape
    window = torch.hann_window(win, device="cuda")
    resid = torch.empty(n, dtype=torch.float64, device="cuda")
    norm_a = torch.empty_like(resid)
    ws = lib().jk_stft_workspace_bytes(n, T, n_fft, hop)
    work = torch.empty(max(ws, 8), dtype=torch.uint8, device="cuda")
    check(lib().jk_stft_mag_diff(ptr(a), ptr(b), ptr(window), ptr(resid), ptr(norm_a), n, T, n_fft, hop, win,
                                 ptr(work), work.numel(), stream_ptr()))
    torch.cuda.synchronize()
    return resid.cpu().numpy(), norm_a.cpu().numpy()


def _check_against_oracle(a, b, cfg, tag):
    """sqrt(norm_a) within rel 1e-5, sqrt(resid) within 1e-5 * sqrt(norm_a); the oracle runs clip by clip"""
    resid, norm_a = _sums(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), *cfg)
    ref = [audio_np.stft_sums(a[i:i + 1], b[i:i + 1], *cfg) for i in range(a.shape[0])]
    ref_r = np.array([r[0][0] for r in ref])
    ref_n = np.array([r[1][0] for r in ref])
    e_norm = float(np.max(np.abs(np.sqrt(norm_a) - np.sqrt(ref_n)) / np.sqrt(ref_n)))
    e_res = float(np.max(np.abs(np.sqrt(resid) - np.sqrt(ref_r)) / np.sqrt(ref_n)))
    print(f"{tag} {cfg}: |sqrt(norm_a)| rel err {e_norm:.2e}, |sqrt(resid)| err / sqrt(norm_a) {e_res:.2e}")
    assert e_norm <= 1e-5 and e_res <= 1e-5, (tag, cfg, e_norm, e_res)


def test_stft_kernel_matches_fp64_oracle_at_c5_geometry():
    rng = np.random.default_rng(5)
    n, T = 16, 1 << 20
    a = (0.3 * rng.standard_normal((n, T))).astype(np.float32)
    pairs = {"independent": (0.3 * rng.standard_normal((n, T))).astype(np.float32),
             "a + 1e-3 noise": (a + 1e-3 * rng.standard_normal((n, T))).astype(np.float32)}
    for tag, b in pairs.items():
        for cfg in CONFIGS:
            _check_against_oracle(a, b, cfg, tag)


@pytest.mark.parametrize("n,T,n_fft,hop,win", [
    (3, 10007, 256, 50, 240),          # smallest n_fft, T not a multiple of hop
    (2, 50000, 4096, 1000, 4096),      # largest n_fft, win_length == n_fft
    (2, 30011, 2048, 240, 601),        # odd win_length
    (1, 1025, 2048, 256, 2048),        # T = n_fft / 2 + 1
    (1, 129, 256, 1, 255),             # hop 1, T = n_fft / 2 + 1
    (1, 3000, 4096, 5000, 3001),       # hop > T: one frame
])
def test_stft_kernel_edge_shapes(n, T, n_fft, hop, win):
    rng = np.random.default_rng(T)
    a = rng.uniform(-1, 1, (n, T)).astype(np.float32)
    b = (0.5 * a + 0.5 * rng.uniform(-1, 1, (n, T))).astype(np.float32)
    _check_against_oracle(a, b, (n_fft, hop, win), "edge")


def test_stft_kernel_is_deterministic_and_batch_independent():
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(16, 200003, device="cuda", generator=g)
    b = a + 0.01 * torch.randn(16, 200003, device="cuda", generator=g)
    for cfg in [(512, 50, 240), (2048, 256, 1536)]:
        r1, n1 = _sums(a, b, *cfg)
        r2, n2 = _sums(a, b, *cfg)
        assert np.array_equal(r1, r2) and np.array_equal(n1, n2)
        r5, n5 = _sums(a[5:6].contiguous(), b[5:6].contiguous(), *cfg)
        assert r5[0] == r1[5] and n5[0] == n1[5]


def test_stft_rejects_bad_input():
    from jukebox_b200.utils.audio_utils import stft_stats
    hps = types.SimpleNamespace
    a = torch.randn(2, 4096, 1, device="cuda")
    with pytest.raises(RuntimeError, match="power of two"):
        stft_stats(a, a, hps(n_fft=1000, hop_length=100, window_size=800))
    with pytest.raises(RuntimeError, match="win_length"):
        stft_stats(a, a, hps(n_fft=1024, hop_length=100, window_size=1025))
    with pytest.raises(RuntimeError, match="reflect padding"):
        stft_stats(a[:, :1024], a[:, :1024], hps(n_fft=2048, hop_length=256, window_size=1536))
    from jukebox_b200.vqvae.bottleneck import BottleneckBlock
    with pytest.raises(NotImplementedError):
        BottleneckBlock(16, 64, 0.99).cuda()(torch.zeros(1, 4, 64, device="cuda"), update_k=True)


def _make(fx):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae
    c = fx.cfg
    hps = setup_hparams(c["hps_name"], dict(restore_vqvae="", **c["overrides"]))
    vq = make_vqvae(hps, "cpu")
    vq.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
    hps.bandwidth = dict(c["bandwidth"])
    return vq.cuda().eval(), hps


def test_forward_in_training_mode_raises():
    fx = Fixture("vqvae_forward_3level")
    vq, hps = _make(fx)
    with pytest.raises(NotImplementedError):
        vq.train()(torch.from_numpy(fx["x"]).cuda(), hps)


CASES = [f"{l}_{s}" for l in ("lmix", "l1", "l2", "linf") for s in ("nonrel", "conv")]


@pytest.mark.parametrize("case", CASES)
def test_forward_matches_reference(case):
    fx = Fixture("vqvae_forward_3level")
    spec = next(c for c in fx.cfg["cases"] if c["case"] == case)
    vq, hps = _make(fx)
    hps.use_nonrelative_specloss = spec["use_nonrelative_specloss"]
    x = torch.from_numpy(fx["x"]).cuda()
    x_out, loss, metrics = vq(x, hps, loss_fn=spec["loss_fn"])
    assert sorted(metrics) == spec["keys"]
    assert all(v.dim() == 0 and not v.requires_grad for v in metrics.values())
    # codes against the reference's (vqvae_3level is the same model and input); a flip only on a near-tie
    enc = Fixture("vqvae_3level")
    assert np.array_equal(enc["x"], fx["x"])
    flips = 0
    with torch.no_grad():
        zs = vq.encode(x)
        lat = [vq.encoders[l](vq.preprocess(x))[-1] for l in range(fx.cfg["levels"])]
    for l in range(fx.cfg["levels"]):
        z, zref = zs[l].cpu().numpy(), enc[f"z{l}"]
        for n, t in np.argwhere(z != zref):
            _, d = quantise(lat[l][n, t:t + 1].cpu().numpy(), fx.weights()[f"bottleneck.level_blocks.{l}.k"])
            assert abs(d[0, z[n, t]] - d[0, zref[n, t]]) < 1e-4 * abs(d[0, zref[n, t]]), (l, n, t)
            flips += 1
    if flips == 0:
        e = rel_err(x_out.cpu().numpy(), fx["x_out"])
        print(f"{case}: x_out rel err {e:.2e}")
        assert e < 2e-5
    worst = 0.0
    for k, v in list(metrics.items()) + [("loss", loss)]:
        ref = float(fx[f"{case}/{k}"])
        err = abs(float(v) - ref) / max(abs(ref), 1e-30)
        worst = max(worst, err)
        assert err <= 1e-4, (case, k, float(v), ref)
    print(f"{case}: {flips} code flips, worst metric rel err {worst:.2e}")
