"""Given rows of a window with fewer given rows than engine rows (no GPU): the prefill and the steps of given positions
read rows [0, n) of the window's tokens, so those rows must hold the n given rows in order before select fans them out -
for packed regeneration (M primes for M x K rows) and for a guided one-row prime with its own alternative x_alt."""
import pytest
import torch

import jukebox_b200.prior.autoregressive as ar
import jukebox_b200.score as score


class FakeEngine:
    """records the token rows the prefill / the given steps read, and follows which given row each engine row holds"""
    has_logits_gemm = False

    def __init__(self, capacity, rows):
        self.prefill_capacity = capacity
        self.rows = list(range(rows))
        self.read = {}          # position -> the tokens at that position of the rows read
        self.position = 0

    def reset(self, t0=0):
        self.position = t0

    def set_encoder_kv(self, kv):
        pass

    def prefill(self, n, P, tokens=None, h_out=None, **kw):
        for p in range(self.position, self.position + P):
            self.read.setdefault(p, tokens[:n, p].clone())
        if h_out is not None:
            h_out.zero_()
        self.position += P

    def step(self, n, tokens=None, logits=None, h_out=None, **kw):
        self.read.setdefault(self.position, tokens[:n, self.position].clone())
        for v in (logits, h_out):
            if v is not None:
                v.zero_()
        self.position += 1

    def select(self, parents):
        self.rows = [self.rows[p] for p in parents]


def _model(monkeypatch, capacity, rows, D=24):
    m = ar.ConditionalAutoregressive2D((D,), 16, width=64, depth=2, heads=1, attn_order=0, blocks=None).eval()
    eng = FakeEngine(capacity, rows)
    monkeypatch.setattr(m, "_engine", lambda n: eng)
    monkeypatch.setattr(m.transformer, "check_cache", lambda *a, **k: None)
    return m, eng


@pytest.mark.parametrize("capacity", [512, 0])
def test_packed_primes_run_on_their_own_rows(monkeypatch, capacity):
    M, K, D, start, end = 4, 8, 24, 5, 9
    m, eng = _model(monkeypatch, capacity, M * K, D)
    monkeypatch.setattr(m, "engine_rows", lambda: 32)

    def fake_sample(logits, temp, seed, position, tokens):
        tokens[:, position] = torch.arange(tokens.shape[0]) % 16
    monkeypatch.setattr(ar, "sample_categorical", fake_sample)
    seen = []
    monkeypatch.setattr(score, "xout_logprob", lambda a, w, tg: (seen.append(tg.clone()), torch.zeros(tg.numel()))[1])
    x = torch.randint(0, 16, (M, D), generator=torch.Generator().manual_seed(0))
    x_new, scores = m.regenerate(x, start, end, K, pack=True)
    for p in range(start):                                  # the given positions ran item i on row i
        assert torch.equal(eng.read[p], x[:, p]), f"position {p}: rows read {eng.read[p].tolist()}"
    assert eng.rows == [b // K for b in range(M * K)]       # then item i's state on rows [i K, (i + 1) K)
    assert torch.equal(seen[0].view(M * K, D - end), x[:, end:].repeat_interleave(K, dim=0))
    for i in range(M):
        assert torch.equal(x_new[i, :start], x[i, :start]) and torch.equal(x_new[i, end:], x[i, end:])


def test_captured_candidate_rows_begin_with_their_own_item(monkeypatch):
    M, K, D, start, end = 3, 4, 24, 6, 10
    m, eng = _model(monkeypatch, 512, M * K, D)
    monkeypatch.setattr(m, "engine_rows", lambda: 32)
    monkeypatch.setattr(ar, "sample_categorical", lambda logits, temp, seed, pos, tokens: None)
    monkeypatch.setattr(score, "xout_logprob", lambda a, w, tg: torch.zeros(tg.numel()))
    rows = []
    orig = ar.ConditionalAutoregressive2D._suffix_acts
    monkeypatch.setattr(ar.ConditionalAutoregressive2D, "_suffix_acts",
                        lambda self, win, e, d: (rows.append(win.tokens.clone()), orig(self, win, e, d))[1])
    x = torch.randint(0, 16, (M, D), generator=torch.Generator().manual_seed(1))
    m.regenerate(x, start, end, K, pack=True)
    assert torch.equal(rows[0][:, :start], x[:, :start].repeat_interleave(K, dim=0))


@pytest.mark.parametrize("capacity", [512, 0])
def test_guided_one_row_prime_runs_its_alternative(monkeypatch, capacity):
    N, P = 3, 4
    m, eng = _model(monkeypatch, capacity, 2 * N)
    monkeypatch.setattr(m, "items_per_prefill", lambda n: min(n, 32))

    def fake_guided(c, u, s, temp, top_k, top_p, seed, position, tokens, tokens_alt, logp=None):
        tokens[:, position] = 1
        tokens_alt[:, position] = 1
    monkeypatch.setattr(ar, "sample_guided", fake_guided)
    prime, x_alt = torch.tensor([[3, 4, 5, 6]]), torch.tensor([[7, 8, 9, 10]])
    wins = []
    orig = ar.SamplingWindow.finish
    monkeypatch.setattr(ar.SamplingWindow, "finish", lambda self: (wins.append(self.tokens.clone()), orig(self))[1])
    z = m.primed_sample(N, prime, fp16=True, sample_tokens=6, guidance_scale=2.0, x_alt=x_alt)
    for p in range(P):
        assert eng.read[p].tolist() == [int(prime[0, p]), int(x_alt[0, p])]
    assert torch.equal(wins[0][:N, :P], prime.expand(N, -1)) and torch.equal(wins[0][N:, :P], x_alt.expand(N, -1))
    assert torch.equal(z[:, :P], prime.expand(N, -1))
