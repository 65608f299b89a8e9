"""CPU checks of token statistics (no GPU): jk_xout_stats / jk_xout_stats_workspace_bytes are declared, exported and
bound, and validate their arguments; the fp64 oracle's entropy and top-k; the host flow of token_stats with the engine
replaced; and the whole-song window plan: the scored positions partition [0, T) and each token is scored in the window
plan_windows gives the sampler for it."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import score_np, stats_np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = {"jk_xout_stats_workspace_bytes": 5, "jk_xout_stats": 15}


def test_stats_symbols_are_declared_exported_and_bound():
    from jukebox_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jkb200.h")).read()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    lib = _lib.lib()
    for name, n_args in NEW.items():
        m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", header)
        assert m, f"{name} not declared"
        assert len(m.group(1).split(",")) == n_args, name
        res, args = _lib.SIGNATURES[name]
        assert res is ctypes.c_int and len(args) == n_args, name
        assert hasattr(handle, name)
        assert getattr(lib, name).argtypes == args
    assert re.search(r"#define\s+JK_XOUT_STATS_MAX_K\s+(\d+)", header).group(1) == str(_lib.JK_XOUT_STATS_MAX_K)


def test_stats_workspace_sizes_and_argument_checks():
    from jukebox_b200 import _lib
    lib = _lib.lib()
    b, b0 = ctypes.c_size_t(0), ctypes.c_size_t(0)
    up = lambda v: (v + 255) // 256 * 256
    for M, W, bins, k in ((1000, 1280, 2048, 16), (300, 4800, 2127, 5), (1, 64, 80, 1), (129, 1920, 128, 0)):
        assert lib.jk_xout_stats_workspace_bytes(M, W, bins, k, ctypes.byref(b)) == 0
        assert lib.jk_xout_logprob_workspace_bytes(M, W, bins, ctypes.byref(b0)) == 0
        slots = M * -(-bins // 128)
        # the logprob layout plus u and the tiles' top-k logits and bins
        assert b.value == b0.value + up(slots * 4) + 2 * up(slots * k * 4), (M, W, bins, k)
    assert lib.jk_xout_stats_workspace_bytes(0, 64, 80, 3, ctypes.byref(b)) == 0
    for args, msg in (((10, 64, 80, 17), b"k <= min"), ((10, 64, 5, 6), b"k <= min"), ((10, 64, 80, -1), b"k <= min"),
                      ((10, 100, 80, 4), b"multiple of 64"), ((-1, 64, 80, 4), b"m >= 0")):
        assert lib.jk_xout_stats_workspace_bytes(*args, ctypes.byref(b)) != 0, args
        assert msg in lib.jk_last_error(), (args, lib.jk_last_error())
    # checks that need no device: null arguments and the pairing of targets with logp
    P = ctypes.c_void_p
    ws = ctypes.c_size_t(1 << 20)
    fake = P(4096)
    call = lambda tg, logp, ent, ids, tlp, k: lib.jk_xout_stats(fake, 10, 64, fake, 80, tg, k, logp, ent, ids, tlp,
                                                              P(0), fake, ws, P(0))
    assert call(P(0), P(0), P(0), P(0), P(0), 0) != 0 and b"null argument" in lib.jk_last_error()
    assert call(fake, P(0), fake, P(0), P(0), 0) != 0 and b"together" in lib.jk_last_error()
    assert call(P(0), P(0), fake, P(0), P(0), 4) != 0 and b"topk_ids" in lib.jk_last_error()
    assert lib.jk_xout_stats(fake, 10, 64, fake, 80, P(0), 0, P(0), fake, P(0), P(0), P(0), fake, ctypes.c_size_t(16),
                             P(0)) != 0
    assert b"workspace of 16 bytes" in lib.jk_last_error()


def test_oracle_entropy_and_topk():
    rng = np.random.RandomState(0)
    z = rng.standard_normal((7, 300)) * 3
    z[0, [5, 17, 250]] = z[0].max() + 1.0            # an exact three-way tie at the top
    p = torch.softmax(torch.from_numpy(z), -1).numpy()
    np.testing.assert_allclose(stats_np.entropy_from_logits(z), -(p * np.log(p)).sum(-1), rtol=1e-12)
    ids, lp = stats_np.topk_from_logits(z, 6)
    assert ids[0, :3].tolist() == [5, 17, 250]
    want = torch.log_softmax(torch.from_numpy(z), -1).topk(6, -1).values.numpy()
    np.testing.assert_allclose(lp, want, atol=1e-12)
    np.testing.assert_allclose(stats_np.entropy_from_logits(np.zeros((2, 64))), np.log(64.0), rtol=1e-14)
    h, w = rng.standard_normal((5, 64)), rng.standard_normal((50, 64)) * 0.1
    t = rng.randint(0, 50, 5)
    lp1, H, ids, tlp, lse, zz = stats_np.xout_stats(h, w, t, 3)
    np.testing.assert_allclose(lp1, score_np.xout_logprob(h, w, t)[0], atol=1e-14)
    assert ids.shape == (5, 3) and tlp.shape == (5, 3) and H.shape == lse.shape == (5,)


# ---- host flow -----------------------------------------------------------------------------------------------------
def test_token_stats_shares_logprob_prefill(monkeypatch):
    """token_stats and logprob read the same activations (one helper); a prefix reads the first D rows of x_cond"""
    import jukebox_b200.prior.autoregressive as ar
    import jukebox_b200.score as score
    m = ar.ConditionalAutoregressive2D((24,), 16, width=64, depth=2, heads=1, attn_order=0, blocks=None,
                                       x_cond=True, y_cond=True).eval()
    seen = []

    def fake_prefill(x, x_cond, y_cond, encoder_kv, h_out=None, **kw):
        seen.append((tuple(x.shape), tuple(x_cond.shape)))
        h_out.copy_(torch.arange(x.shape[1], dtype=torch.float)[None, :, None].expand(x.shape[0], x.shape[1], 64))
    got = {}

    def fake_stats(h, w, targets=None, top_k=0):
        got["h"], got["t"], got["k"] = h.clone(), targets.clone(), top_k
        M = h.shape[0]
        return score.TokenStats(torch.zeros(M), torch.ones(M), torch.zeros(M, top_k, dtype=torch.long),
                                torch.zeros(M, top_k), torch.zeros(M))

    def fake_logprob(h, w, targets):
        got["h_lp"] = h.clone()
        return torch.zeros(h.shape[0])
    monkeypatch.setattr(m, "_prefill", fake_prefill)
    monkeypatch.setattr(score, "xout_stats", fake_stats)
    monkeypatch.setattr(score, "xout_logprob", fake_logprob)
    x = torch.randint(0, 16, (2, 24))
    xc = torch.randn(2, 24, 64)
    yc = torch.randn(2, 1, 64)
    m.logprob(x, xc, yc)
    st = m.token_stats(x, xc, yc, top_k=3)
    assert torch.equal(got["h"], got["h_lp"]) and got["k"] == 3
    assert st.entropy.shape == (2, 24) and st.topk_ids.shape == (2, 24, 3)
    st = m.token_stats(x[:, :10], xc, yc)
    assert seen[-1] == ((2, 10), (2, 24, 64))
    want = (torch.arange(10, dtype=torch.float)[None, :, None] + xc[:, :10]).reshape(20, 64)
    assert torch.equal(got["h"], want) and torch.equal(got["t"], x[:, :10].reshape(-1))
    with pytest.raises(AssertionError):
        m.token_stats(x[:, :1], xc, yc)


# ---- the whole-song plan -----------------------------------------------------------------------------------------
def _sampler_windows(T, n_ctx, hop):
    """for each token, the window (start, length) in which LevelRun.extend_to(T) draws it from an empty level"""
    from jukebox_b200.sample import plan_windows
    owner, have = {}, 0
    for win in plan_windows(0, T, n_ctx, hop):
        end = win.start + win.sample_tokens
        for tok in range(have, end):
            owner[tok] = (win.start, win.sample_tokens)
        have = max(have, end)
    return owner


@pytest.mark.parametrize("n_ctx,hop_fraction", [(8192, 0.5), (6144, 0.125), (8192, 0.125), (64, 0.5), (64, 0.25)])
def test_song_windows_partition_and_match_the_sampler(n_ctx, hop_fraction):
    """hop fractions of the sampling presets: 0.5 at the upsampler levels, 0.125 at the top level (n_ctx 6144 / 8192)"""
    from jukebox_b200.sample import song_windows
    hop = int(hop_fraction * n_ctx)
    for T in (2, n_ctx // 3, n_ctx - 1, n_ctx, n_ctx + 1, 2 * n_ctx, 3 * n_ctx + hop // 3, 5 * n_ctx - 7):
        plan = song_windows(T, n_ctx, hop)
        spans = [(t0, t1) for _, t0, t1 in plan]
        assert spans[0][0] == 0 and spans[-1][1] == T and all(a[1] == b[0] for a, b in zip(spans, spans[1:])), (T, spans)
        assert all(t0 < t1 for t0, t1 in spans)
        owner = _sampler_windows(T, n_ctx, hop)
        for win, t0, t1 in plan:
            assert win.start <= t0 and t1 <= win.start + min(n_ctx, win.sample_tokens)
            for tok in (t0, (t0 + t1) // 2, t1 - 1):
                assert owner[tok] == (win.start, win.sample_tokens), (T, tok)


class _FakePrior:
    """records what song_token_stats asks for: the window's context, labels start and upper-level span"""
    def __init__(self, n_ctx, ds):
        self.n_ctx, self.cond_downsample, self.calls = n_ctx, ds, []

    def get_z_conds(self, zs, start, end):
        return [zs[1][:, start // self.cond_downsample:end // self.cond_downsample]]

    def get_y(self, labels, start):
        return labels["y"] + start

    def token_stats(self, z, z_conds, y, fp16=True, top_k=0):
        from jukebox_b200.score import TokenStats
        self.calls.append((tuple(z.shape), int(z_conds[0][0, 0]), int(y[0, 0]), top_k))
        N, D = z.shape
        return TokenStats(z.float(), -z.float(), None, None, torch.zeros(N, D))


def test_song_token_stats_scores_each_token_in_its_window():
    from jukebox_b200.sample import song_token_stats, plan_windows
    n_ctx, hop, ds, N, T = 16, 8, 4, 5, 44
    prior = _FakePrior(n_ctx, ds)
    z = torch.arange(T)[None].repeat(N, 1)
    zs = [z, torch.arange(T // ds + n_ctx)[None].repeat(N, 1)]
    labels = dict(y=torch.zeros(N, 3, dtype=torch.long))
    st = song_token_stats(prior, zs, labels, 0, hop, max_batch_size=2)
    assert torch.equal(st.logp, z.float()) and torch.equal(st.entropy, -z.float()) and st.topk_ids is None
    starts = [w.start for w in plan_windows(0, T, n_ctx, hop)]
    # per window three pieces of the batch (2 + 2 + 1), each with the window's labels and upper-level codes
    assert [c[2] for c in prior.calls] == [s for s in starts for _ in range(3)]
    assert [c[1] for c in prior.calls] == [s // ds for s in starts for _ in range(3)]
    assert [c[0][0] for c in prior.calls] == [2, 2, 1] * len(starts)
