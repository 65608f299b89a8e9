"""Regenerating a section (no GPU): the window regen_window places, and the host-side call sequence of
ConditionalAutoregressive2D.regenerate with the engine, the sampler and the scoring kernel replaced by recorders -
one-row prime prefill, one broadcast, the span's steps, ONE continuation prefill of the kept codes, nothing after."""
import pytest
import torch

import jukebox_b200.prior.autoregressive as ar
import jukebox_b200.score as score
from jukebox_b200.sample import regen_window


# ---- regen_window -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T, start, end, n_ctx, want", [
    (100, 2, 5, 10, (0, 10)),          # near the start: clamped to 0
    (100, 50, 54, 10, (47, 57)),       # middle: (10 - 4) // 2 = 3 codes before, 3 after
    (100, 50, 55, 10, (48, 58)),       # odd remainder: the extra code goes after the span
    (100, 95, 98, 10, (90, 100)),      # near the end: clamped to T - n_ctx
    (100, 0, 9, 10, (0, 10)),          # the longest span at the head
    (100, 90, 99, 10, (90, 100)),      # the longest span at the tail
    (7, 2, 4, 10, (0, 7)),             # a level shorter than n_ctx: the whole level
    (7, 0, 6, 10, (0, 7)),
])
def test_regen_window_places_the_span(T, start, end, n_ctx, want):
    w0, w1 = regen_window(T, start, end, n_ctx)
    assert (w0, w1) == want
    assert w0 <= start and end < w1 and w1 - w0 <= n_ctx and w1 <= T


def test_regen_window_every_placement_keeps_a_suffix():
    for T in (5, 17, 40):
        for n_ctx in (4, 9, 16):
            for start in range(T):
                for end in range(start + 1, min(T, start + n_ctx)):
                    w0, w1 = regen_window(T, start, end, n_ctx)
                    assert 0 <= w0 <= start < end < w1 <= T and w1 - w0 == min(T, n_ctx)


@pytest.mark.parametrize("T, start, end, n_ctx", [
    (100, 5, 5, 10),        # empty span
    (100, 6, 5, 10),        # reversed
    (100, 95, 100, 10),     # end == T: no codes after it
    (100, 95, 101, 10),     # past the level
    (100, 10, 20, 10),      # span as long as the context
    (100, 10, 25, 10),
    (100, -1, 3, 10),
])
def test_regen_window_errors(T, start, end, n_ctx):
    with pytest.raises(ValueError):
        regen_window(T, start, end, n_ctx)


# ---- call sequence ---------------------------------------------------------------------------------------------------------
class FakeEngine:
    has_logits_gemm = False

    def __init__(self, capacity):
        self.prefill_capacity = capacity
        self.calls = []
        self.position = 0

    def reset(self, t0=0):
        self.position = t0

    def set_encoder_kv(self, kv):
        self.calls.append(("enc", tuple(kv.shape)))

    def prefill(self, n, P, h_out=None, tokens=None, **kw):
        self.calls.append(("prefill", n, P, self.position))
        if h_out is not None:
            h_out.zero_()
        self.position += P

    def step(self, n, tokens=None, logits=None, h_out=None, **kw):
        self.calls.append(("step", n, self.position))
        if logits is not None:
            logits.zero_()
        if h_out is not None:
            h_out.zero_()
        self.position += 1

    def select(self, parents):
        self.calls.append(("select", list(parents)))


def _model(monkeypatch, capacity, D=24):
    m = ar.ConditionalAutoregressive2D((D,), 16, width=64, depth=2, heads=1, attn_order=0, blocks=None).eval()
    eng = FakeEngine(capacity)
    monkeypatch.setattr(m, "_engine", lambda n: eng)
    monkeypatch.setattr(m.transformer, "check_cache", lambda *a, **k: None)
    drawn = []

    def fake_sample(logits, temp, seed, position, tokens):
        drawn.append((tokens.shape[0], position))
        tokens[:, position] = torch.arange(tokens.shape[0]) % 16       # candidate c draws code c
    monkeypatch.setattr(ar, "sample_categorical", fake_sample)
    scored = []

    def fake_logprob(acts, w, targets):
        scored.append((tuple(acts.shape), targets.clone()))
        return -torch.arange(targets.numel(), dtype=torch.float32).remainder(5)   # unequal candidates' scores
    monkeypatch.setattr(score, "xout_logprob", fake_logprob)
    return m, eng, drawn, scored


@pytest.mark.parametrize("start, end", [(7, 12), (1, 3), (0, 4)])
def test_one_item_prefills_the_suffix_once(monkeypatch, start, end):
    D, K = 24, 4
    m, eng, drawn, scored = _model(monkeypatch, capacity=512, D=D)
    x = torch.randint(0, 16, (1, D))
    x_new, scores = m.regenerate(x, start, end, K)
    calls = eng.calls
    i = 0
    if start > 1:       # a one-row prefill of the prime (one given position is stepped on its row)
        assert calls[0] == ("prefill", 1, start, 0)
        i = 1
    elif start == 1:
        assert calls[0] == ("step", 1, 0)
        i = 1
    if start:
        assert calls[i][0] == "select" and calls[i][1] == [0] * K           # one broadcast
        i += 1
    steps = calls[i:i + end - start]
    assert steps == [("step", K, p) for p in range(start, end)]
    assert calls[i + end - start:] == [("prefill", K, D - end, end)]        # one continuation prefill, nothing after
    assert [p for _, p in drawn] == list(range(start, end))
    assert len(scored) == 1 and scored[0][0] == (K * (D - end), 64)
    assert torch.equal(scored[0][1].view(K, D - end), x[0, end:].expand(K, -1))   # the kept codes are what is scored
    assert scores.shape == (1, K) and scores.dtype == torch.float32
    best = int(torch.argmax(scores[0]))
    assert torch.equal(x_new[0, :start], x[0, :start]) and torch.equal(x_new[0, end:], x[0, end:])
    assert bool((x_new[0, start:end] == best % 16).all())


def test_without_capacity_the_suffix_is_stepped(monkeypatch):
    D, K, start, end = 24, 3, 6, 10
    m, eng, drawn, scored = _model(monkeypatch, capacity=0, D=D)
    x = torch.randint(0, 16, (2, D))
    x_new, scores = m.regenerate(x, start, end, K)
    per_item = len(eng.calls) // 2
    calls = eng.calls[:per_item]
    assert all(c[0] != "prefill" for c in eng.calls)
    assert calls[:start] == [("step", 1, p) for p in range(start)] and calls[start] == ("select", [0] * K)
    assert calls[start + 1:] == [("step", K, p) for p in range(start, D)]
    assert scores.shape == (2, K) and len(scored) == 2


def test_ties_go_to_the_lower_candidate_and_errors(monkeypatch):
    D = 24
    m, eng, drawn, scored = _model(monkeypatch, capacity=512, D=D)
    monkeypatch.setattr(score, "xout_logprob", lambda a, w, tg: torch.zeros(tg.numel()))
    x = torch.randint(0, 16, (1, D))
    x_new, scores = m.regenerate(x, 3, 8, 5)
    assert bool((scores == 0).all()) and bool((x_new[0, 3:8] == 0).all())
    for bad in ((3, 24), (5, 5), (8, 3), (-1, 4)):
        with pytest.raises(ValueError):
            m.regenerate(x, *bad, 4)
    with pytest.raises(ValueError):
        m.regenerate(x, 3, 8, 0)
