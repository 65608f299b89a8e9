"""CPU checks of token scoring (no GPU): the new C entries are declared, exported and bound with their ctypes
signatures; the fp64 scoring oracle reproduces log-softmax-at-target and the loss of the golden fixtures' fp32
logits; and the host control flow of sample(get_logprobs=True) - which positions are scored, from which logits,
through which launch - with the engine and the kernels replaced by recorders."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import jukebox_b200.prior.autoregressive as ar
from golden_util import Fixture
from oracle import score_np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = {
    "jk_sample_categorical_scored": 14,
    "jk_xout_split_bytes": 3,
    "jk_pack_xout_split": 5,
    "jk_xout_logprob_workspace_bytes": 4,
    "jk_xout_logprob": 11,
}


def test_scoring_symbols_are_declared_exported_and_bound():
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
    # the sizes need no device
    b = ctypes.c_size_t(0)
    assert lib.jk_xout_split_bytes(2127, 2048, ctypes.byref(b)) == 0
    assert b.value == 2 * 17 * 128 * 2048 * 2 + 16                     # [hi | lo][bins padded to 128][W] fp16 + status
    assert lib.jk_xout_split_bytes(80, 1000, ctypes.byref(b)) != 0      # width not a multiple of 64
    assert b"multiple of 64" in lib.jk_last_error()
    assert lib.jk_xout_logprob_workspace_bytes(1000, 1280, 2048, ctypes.byref(b)) == 0
    assert b.value >= 1000 * 16 * 8 + 1000 * 4


@pytest.mark.parametrize("tag", ["ca2d_xy", "ca2d_plain", "ca2d_encdec_merged"])
def test_oracle_logprob_of_golden_logits(tag):
    fx = Fixture(tag)
    z, tok = fx["preds32"], fx["tokens"]
    lp = score_np.logprob_from_logits(z, tok)
    want = torch.log_softmax(torch.from_numpy(z).double(), -1).gather(-1, torch.from_numpy(tok)[..., None])[..., 0]
    np.testing.assert_allclose(lp, want.numpy(), rtol=0, atol=1e-12)
    bits = score_np.bits_per_token(lp)
    loss = F.cross_entropy(torch.from_numpy(z).double().reshape(-1, z.shape[-1]), torch.from_numpy(tok).reshape(-1))
    assert abs(bits.mean() - float(loss) / np.log(2.0)) < 1e-12
    # from activations: h . w^T gives the same as the logits it makes
    rng = np.random.RandomState(0)
    h, w = rng.standard_normal((5, 64)), rng.standard_normal((50, 64)) * 0.1
    t = rng.randint(0, 50, 5)
    lp2, lse = score_np.xout_logprob(h, w, t)
    np.testing.assert_allclose(lp2, score_np.logprob_from_logits(h @ w.T, t), atol=1e-12)
    np.testing.assert_allclose(np.exp(lp2), torch.softmax(torch.from_numpy(h @ w.T), -1).numpy()[np.arange(5), t],
                               rtol=1e-12)
    assert lse.shape == (5,)


# ---- control flow of get_logprobs ------------------------------------------------------------------------------------
class FakeEngine:
    def __init__(self, capacity):
        self.prefill_capacity = capacity
        self.has_logits_gemm = False
        self.calls = []
        self.position = 0

    def reset(self, t0=0):
        self.position = t0

    def prefill(self, n, P, h_out=None, **kw):
        self.calls.append(("prefill", n, P, None if h_out is None else tuple(h_out.shape)))
        if h_out is not None:
            h_out.zero_()
        self.position = P

    def step(self, n, tokens=None, logits=None, **kw):
        self.calls.append(("step", self.position, logits is not None))
        if logits is not None:
            (logits[:, self.position] if logits.dim() == 3 else logits).fill_(float(self.position))
        self.position += 1


def _model(monkeypatch, capacity):
    import jukebox_b200.score as score
    m = ar.ConditionalAutoregressive2D((24,), 16, width=64, depth=2, heads=1, attn_order=0, blocks=None).eval()
    eng = FakeEngine(capacity)
    monkeypatch.setattr(m, "_engine", lambda n: eng)
    monkeypatch.setattr(m.transformer, "check_cache", lambda *a, **k: None)
    rec = dict(plain=[], scored=[], xout=[], filt=[])

    def fake_sample(logits, temp, seed, position, tokens):
        rec["plain"].append(position)
        tokens[:, position] = position % 16

    def fake_scored(logits, raw, temp, seed, position, tokens, logp):
        rec["scored"].append((position, None if logits is None else float(logits[0, 0]), float(raw[0, 0]), temp))
        if logits is not None:
            tokens[:, position] = position % 16
        logp[:, position] = -float(position)

    def fake_filter(x, temp, top_k, top_p, out):
        rec["filt"].append(float(x[0, 0]))
        return x * 0 - 1.0                      # the sampler then sees -1: distinguishes it from the raw row

    def fake_xout(h, w, targets):
        rec["xout"].append((tuple(h.shape), tuple(w.shape), targets.tolist()))
        return torch.full((h.shape[0],), -0.5)
    monkeypatch.setattr(ar, "sample_categorical", fake_sample)
    monkeypatch.setattr(ar, "sample_categorical_scored", fake_scored)
    monkeypatch.setattr(ar, "filter_logits_scaled", fake_filter)
    monkeypatch.setattr(score, "xout_logprob", fake_xout)
    return m, eng, rec


def test_stepped_given_positions_are_scored_from_the_engine_logits(monkeypatch):
    m, eng, rec = _model(monkeypatch, capacity=0)
    prime = torch.randint(0, 16, (2, 7))
    z, lp = m.primed_sample(2, prime, fp16=True, temp=0.9, sample_tokens=10, get_logprobs=True)
    assert all(c[0] == "step" for c in eng.calls)
    assert [c[2] for c in eng.calls] == [True] * 10                      # logits wanted at given positions too
    # given positions: no draw, scored against the step's raw logits; drawn: draw + score in one launch
    assert rec["scored"] == [(t, None, float(t), 0.9) for t in range(7)] + [(t, float(t), float(t), 0.9) for t in range(7, 10)]
    assert rec["plain"] == [] and rec["xout"] == []
    assert torch.equal(z[:, :7], prime) and lp.shape == (2, 10)
    assert lp[0].tolist() == [-float(t) for t in range(10)]
    # without get_logprobs the given positions keep their logits-free steps and the unscored draw
    m, eng, rec = _model(monkeypatch, capacity=0)
    z = m.primed_sample(2, prime, fp16=True, temp=0.9, sample_tokens=10)
    assert [c[2] for c in eng.calls] == [t >= 7 for t in range(10)]
    assert rec["plain"] == [7, 8, 9] and rec["scored"] == []


def test_prefilled_given_positions_are_scored_from_the_prefill_activations(monkeypatch):
    import jukebox_b200.transformer.f32 as f32
    m, eng, rec = _model(monkeypatch, capacity=512)
    monkeypatch.setattr(f32, "linear_nk", lambda x, w: torch.full((x.shape[0], w.shape[0]), 7.0))
    prime = torch.randint(0, 16, (2, 7))
    z, preds, lp = m.primed_sample(2, prime, fp16=True, sample_tokens=10, get_preds=True, get_logprobs=True)
    assert eng.calls[0] == ("prefill", 2, 7, (2, 7, 64))
    assert rec["xout"] == [((14, 64), (16, 64), prime.reshape(-1).tolist())]
    assert [r[0] for r in rec["scored"]] == [7, 8, 9]
    assert lp[:, :7].eq(-0.5).all() and lp[0, 7:].tolist() == [-7.0, -8.0, -9.0]
    assert preds.shape == (2, 10, 16)


def test_filtered_draw_scores_the_raw_logits(monkeypatch):
    m, eng, rec = _model(monkeypatch, capacity=512)
    z, lp = m.sample(2, fp16=True, temp=0.7, top_k=3, sample_tokens=4, get_logprobs=True)
    # the draw reads the filtered row at temperature 1, the score the raw row
    assert rec["scored"] == [(t, -1.0, float(t), 1.0) for t in range(4)]
    assert rec["filt"] == [float(t) for t in range(4)]
    assert z.shape == (2, 4) and lp.shape == (2, 4)
