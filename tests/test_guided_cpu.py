"""Guided sampling without a GPU: the C ABI of jk_sample_guided and its argument refusals (fake addresses, no launch);
the host flow of a guided window with a fake engine (2N rows stepped, one guided launch per drawn position, scored
launches on given positions, pairs kept together by selection and by a one-row prime's fan-out); the null labels; the
guidance labels windowed by LevelRun; and the refusals of oversized batches and of guided regeneration."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import jukebox_b200.prior.autoregressive as ar
from jukebox_b200 import _lib
from jukebox_b200.data.labels import EmptyLabeller, Labeller
from jukebox_b200.prior.prior import SimplePrior

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_P, _I, _L, _F = C.c_void_p, C.c_int, C.c_int64, C.c_float


# ---- C ABI --------------------------------------------------------------------------------------------------------
def test_guided_symbol_signature():
    want = [_P, _L, _P, _L, _I, _I, _F, _F, _I, _F, C.c_uint64, _I, _P, _L, _P, _L, _P, _P, _L, _P]
    assert _lib.SIGNATURES["jk_sample_guided"] == (_I, want)
    assert len(want) == 20
    assert _lib.lib().jk_sample_guided.argtypes == want
    src = open(os.path.join(ROOT, "include", "jkb200.h")).read()
    decl = re.search(r"int jk_sample_guided\((.*?)\);", src, re.S).group(1)
    assert len(decl.split(",")) == len(want)


def _call(**kw):
    a = dict(c=0x1000, cs=128, u=0x2000, us=128, n=4, bins=80, s=1.0, temp=1.0, top_k=0, top_p=0.0, seed=7, pos=3,
             tok=0x3000, ts=16, alt=0x4000, alts=16, raw=0, logp=0, ls=0)
    a.update(kw)
    lib = _lib.lib()
    rc = lib.jk_sample_guided(_P(a["c"]), a["cs"], _P(a["u"]), a["us"], a["n"], a["bins"], a["s"], a["temp"],
                              a["top_k"], a["top_p"], C.c_uint64(a["seed"]), a["pos"], _P(a["tok"]), a["ts"],
                              _P(a["alt"]), a["alts"], _P(a["raw"]), _P(a["logp"]), a["ls"], _P(0))
    return rc, lib.jk_last_error().decode()


@pytest.mark.parametrize("kw, msg", [
    (dict(c=0), "null"), (dict(u=0), "null"), (dict(tok=0), "null"), (dict(alt=0), "null"),
    (dict(raw=0x5000), "both"), (dict(logp=0x5000), "both"),
    (dict(bins=0), "bins"), (dict(bins=4097), "bins"),
    (dict(temp=0.0), "temp"), (dict(temp=-1.0), "temp"),
    (dict(s=float("inf")), "finite"), (dict(s=float("nan")), "finite"), (dict(s=-float("inf")), "finite"),
    (dict(top_k=4, top_p=0.9), "at most one"), (dict(top_k=-1), "top_k"), (dict(top_p=1.5), "top_p"),
    (dict(n=-1), "negative"), (dict(pos=-1), "negative position"),
])
def test_guided_refuses_bad_arguments_before_any_launch(kw, msg):
    rc, err = _call(**kw)
    assert rc != 0 and msg in err, (kw, err)


def test_guided_with_no_pairs_is_a_no_op():
    # valid arguments and n = 0 return before any CUDA call, so the fake addresses are never touched
    for kw in (dict(), dict(top_k=5), dict(top_p=0.5), dict(raw=0x1000, logp=0x5000, ls=16), dict(s=-0.5)):
        assert _call(n=0, **kw)[0] == 0


# ---- host flow with a fake engine -----------------------------------------------------------------------------------
class FakeEngine:
    """rows carry a label: the row they were first prefilled / stepped as, permuted by select"""

    def __init__(self, capacity, rows):
        self.prefill_capacity = capacity
        self.has_logits_gemm = False
        self.calls = []
        self.position = 0
        self.rows = list(range(rows))

    def set_encoder_kv(self, enc):
        self.calls.append(("enc", enc.shape[0]))

    def prefill(self, n, P, **kw):
        self.calls.append(("prefill", n, P))
        self.position = P

    def step(self, n, tokens=None, y_cond=None, logits=None, **kw):
        self.calls.append(("step", n, self.position))
        if logits is not None:
            logits.zero_()
        self.position += 1

    def select(self, parents):
        self.calls.append(("select", list(parents)))
        self.rows = [self.rows[p] for p in parents]


def _model(monkeypatch, capacity, items, score=lambda r: -1.0, per_prefill=32, y_cond=False):
    m = ar.ConditionalAutoregressive2D((24,), 16, width=64, depth=2, heads=1, attn_order=0, blocks=None,
                                       y_cond=y_cond).eval()
    eng = FakeEngine(capacity, 2 * items)
    log = dict(guided=[], scored=[])
    monkeypatch.setattr(m, "_engine", lambda n: eng)
    monkeypatch.setattr(m, "items_per_prefill", lambda N: min(N, per_prefill))
    monkeypatch.setattr(m.transformer, "check_cache", lambda *a, **k: None)

    def fake_guided(c, u, s, temp, top_k, top_p, seed, position, tokens, tokens_alt, logp=None):
        k = tokens.shape[0]
        assert c.shape[0] == u.shape[0] == tokens_alt.shape[0] == k == len(eng.rows) // 2
        log["guided"].append((position, s, None if logp is None else logp.shape[0]))
        tokens[:, position] = torch.tensor(eng.rows[:k]) % 15 + 1    # a pair draws its conditional row's label
        tokens_alt[:, position] = tokens[:, position]
        if logp is not None:
            logp[:, position] = torch.tensor([score(r) for r in eng.rows[:k]])

    def fake_scored(logits, raw, temp, seed, position, tokens, logp):
        assert logits is None, "a guided window draws through sample_guided"
        log["scored"].append((position, raw.shape[0]))
        logp[:, position] = torch.tensor([score(r) for r in eng.rows[:raw.shape[0]]])
    monkeypatch.setattr(ar, "sample_guided", fake_guided)
    monkeypatch.setattr(ar, "sample_categorical_scored", fake_scored)
    monkeypatch.setattr(ar, "sample_categorical", lambda *a: pytest.fail("a guided window draws through sample_guided"))
    monkeypatch.setattr(ar, "filter_logits_scaled", lambda *a: pytest.fail("the guided launch filters"))
    import jukebox_b200.score as score_mod
    monkeypatch.setattr(score_mod, "xout_logprob", lambda h, w, targets: torch.full((h.shape[0],), -1.0))
    return m, eng, log


def test_guided_window_steps_2n_rows_and_draws_once_per_position(monkeypatch):
    N = 3
    m, eng, log = _model(monkeypatch, 512, N)
    z = m.sample(N, fp16=True, sample_tokens=5, guidance_scale=3.0, top_k=4)
    assert [c for c in eng.calls if c[0] == "step"] == [("step", 2 * N, p) for p in range(5)]
    assert log["guided"] == [(p, 2.0, None) for p in range(5)] and not log["scored"]
    assert z.shape == (N, 5) and z.tolist() == [[1] * 5, [2] * 5, [3] * 5]


@pytest.mark.parametrize("capacity", [512, 0])
def test_given_positions_are_teacher_forced_per_row_and_scored(monkeypatch, capacity):
    N, P = 2, 3
    m, eng, log = _model(monkeypatch, capacity, N)
    prime = torch.tensor([[1, 2, 3], [4, 5, 6]])
    x_alt = torch.tensor([[7, 8, 9], [10, 11, 12]])
    seen = []
    real_init = ar._Rows._init_rows

    def spy(self, *a, **k):
        out = real_init(self, *a, **k)
        seen.append(self.tokens.clone())
        return out
    monkeypatch.setattr(ar._Rows, "_init_rows", spy)
    z, lp = m.primed_sample(N, prime, fp16=True, sample_tokens=6, get_logprobs=True, guidance_scale=0.5, x_alt=x_alt)
    assert torch.equal(seen[0][:N, :P], prime) and torch.equal(seen[0][N:, :P], x_alt)
    if capacity:
        assert eng.calls[0] == ("prefill", 2 * N, P)
        assert [c for c in eng.calls if c[0] == "step"] == [("step", 2 * N, p) for p in range(P, 6)]
    else:     # stepped given positions: each scored on every row, no draw
        assert [c for c in eng.calls if c[0] == "step"] == [("step", 2 * N, p) for p in range(6)]
        assert log["scored"] == [(p, 2 * N) for p in range(P)]
    assert log["guided"] == [(p, -0.5, N) for p in range(P, 6)]
    assert torch.equal(z[:, :P], prime) and lp.shape == (N, 6)


def test_keep_best_moves_pairs_together(monkeypatch):
    N, k, keep = 4, 2, 3
    m, eng, log = _model(monkeypatch, 512, N, score=lambda r: -float(r % N))   # a pair drawn as label r scores -r
    prime = torch.arange(N * 3).view(N, 3) % 16
    z, lp, anc = m.primed_sample(N, prime, fp16=True, sample_tokens=7, get_logprobs=True, select_every=k,
                                 select_keep=keep, guidance_scale=2.0)
    sels = [c[1] for c in eng.calls if c[0] == "select"]
    # the unguided window of test_select_cpu's keep-best test, with each item's parents repeated for its alternative row
    assert sels == [[0, 1, 2, 0, 4, 5, 6, 4], [0, 1, 0, 3, 4, 5, 4, 7]]
    assert eng.rows == [0, 1, 0, 0, 4, 5, 4, 4]
    assert anc.tolist() == [0, 1, 0, 0]
    assert z[:, 3:].tolist() == [[1] * 4, [2] * 4, [1] * 4, [1] * 4]
    assert lp.shape == (N, 7)


@pytest.mark.parametrize("capacity", [512, 0])
def test_one_row_prime_fans_out_to_pairs(monkeypatch, capacity):
    N = 3
    m, eng, log = _model(monkeypatch, capacity, N)
    prime = torch.tensor([[3, 4, 5, 6]])
    z = m.primed_sample(N, prime, fp16=True, sample_tokens=6, guidance_scale=2.0, x_alt=torch.tensor([[1, 1, 1, 1]]))
    if capacity:
        assert eng.calls[0] == ("prefill", 2, 4)
    else:
        assert [c for c in eng.calls if c[0] == "step"][:4] == [("step", 2, t) for t in range(4)]
    i = eng.calls.index(("select", [0] * N + [1] * N))
    assert [c for c in eng.calls[i + 1:]] == [("step", 2 * N, 4), ("step", 2 * N, 5)]
    assert torch.equal(z[:, :4], prime.repeat(N, 1)) and z.shape == (N, 6)


def test_unguided_window_makes_todays_launches(monkeypatch):
    m, eng, log = _model(monkeypatch, 512, 2)
    drawn = []
    monkeypatch.setattr(ar, "sample_categorical", lambda logits, temp, seed, pos, tokens: drawn.append(tokens.shape[0]))
    monkeypatch.setattr(ar, "sample_guided", lambda *a, **k: pytest.fail("no guidance asked"))
    m.sample(4, fp16=True, sample_tokens=3)
    assert drawn == [4, 4, 4]
    assert [c for c in eng.calls if c[0] == "step"] == [("step", 4, p) for p in range(3)]


def test_guided_window_limits_and_conditioning_checks(monkeypatch):
    m, eng, log = _model(monkeypatch, 512, 17)
    with pytest.raises(ValueError, match="at most 16 guided items"):
        m.sample(17, fp16=True, sample_tokens=3, guidance_scale=2.0)
    eng.rows = list(range(32))
    m.sample(16, fp16=True, sample_tokens=2, guidance_scale=2.0)
    monkeypatch.setattr(m, "items_per_prefill", lambda N: min(N, 16))            # an engine of 16 rows (5b_lyrics)
    with pytest.raises(ValueError, match="at most 8 guided items"):
        m.sample(9, fp16=True, sample_tokens=3, guidance_scale=2.0)
    with pytest.raises(ValueError, match="finite"):
        m.sample(2, fp16=True, sample_tokens=3, guidance_scale=float("inf"))
    with pytest.raises(ValueError, match="x_alt"):
        m.primed_sample(2, torch.zeros(2, 3, dtype=torch.long), fp16=True, sample_tokens=5, guidance_scale=2.0,
                        x_alt=torch.zeros(2, 2, dtype=torch.long))
    my = ar.ConditionalAutoregressive2D((24,), 16, width=64, depth=2, heads=1, attn_order=0, blocks=None,
                                        y_cond=True).eval()
    monkeypatch.setattr(my, "items_per_prefill", lambda N: N)
    y = torch.zeros(2, 1, 64)
    with pytest.raises(ValueError, match="y_cond_alt must be given"):
        my.sample(2, y_cond=y, fp16=True, sample_tokens=3, guidance_scale=2.0)
    with pytest.raises(ValueError, match="shape"):
        my.sample(2, y_cond=y, fp16=True, sample_tokens=3, guidance_scale=2.0, y_cond_alt=torch.zeros(1, 1, 64))


# ---- labels ------------------------------------------------------------------------------------------------------
class _LabelPrior:
    """what the label paths of SimplePrior / LevelRun read, with a real Labeller"""
    get_y, null_y = SimplePrior.get_y, SimplePrior.null_y
    n_ctx, level, raw_to_tokens = 8, 0, 4

    def __init__(self, genres=1, n_tokens=12, v3=True, limit=16):
        self.sample_length = self.n_ctx * self.raw_to_tokens
        self.labeller = Labeller(genres, n_tokens, self.sample_length, v3=v3) if genres else EmptyLabeller()
        self.limit, self.calls = limit, []

    def guided_items(self):
        return self.limit

    def get_z_conds(self, zs, start, end):
        return None

    def sample(self, n_samples, z, z_conds, y, **kw):
        self.calls.append((y.clone(), None if kw.get("guidance_y") is None else kw["guidance_y"].clone(),
                           kw.get("guidance_scale")))
        return torch.cat([z, torch.full((n_samples, self.n_ctx - z.shape[1]), 5)], 1)


def _labels(prior, metas):
    return prior.labeller.get_batch_labels(metas, "cpu")


@pytest.mark.parametrize("genres, v3", [(1, True), (5, False)])
def test_null_labels_are_the_labellers_unknown_row(genres, v3):
    from jukebox_b200.sample import null_labels
    prior = _LabelPrior(genres, 12, v3)
    metas = [dict(artist="x", genre="y", lyrics="some words here and more", total_length=320, offset=16 * i)
             for i in range(3)]
    labels = _labels(prior, metas)
    null = null_labels(prior, labels)
    for i, meta in enumerate(metas):
        want = prior.labeller.get_label("unknown", "unknown", "", meta["total_length"], meta["offset"])["y"]
        assert null["y"][i].tolist() == want.tolist()
    assert torch.equal(null["y"][:, :3], labels["y"][:, :3])
    # artist 0, genre 0 then padding, lyric tokens 0
    assert null["y"][0, 3:4 + genres].tolist() == [0, 0] + [-1] * (genres - 1) and not null["y"][:, 4 + genres:].any()
    assert [d["full_tokens"] for d in null["info"]] == [[], [], []]
    with pytest.raises(ValueError, match="no labels"):
        null_labels(_LabelPrior(genres=0), None)


def test_level_run_windows_the_guidance_labels_with_their_lyrics():
    from jukebox_b200.sample import LevelRun, Window
    prior = _LabelPrior()
    N = 4
    words = " ".join(f"line {i}" for i in range(40))
    labels = _labels(prior, [dict(artist="a", genre="b", lyrics="la " * 40, total_length=64, offset=0)] * N)
    guide = _labels(prior, [dict(artist="c", genre="d", lyrics=words, total_length=64, offset=0)] * N)
    zs = [torch.zeros(N, 0, dtype=torch.long)]
    run = LevelRun(zs, labels, dict(max_batch_size=3, guidance_scale=2.5, guidance_labels=guide), 0, prior, None)
    run.extend_to(16, 8)
    assert [c[2] for c in prior.calls] == [2.5] * 4 and zs[0].shape == (N, 16)
    for w, start in enumerate((0, 8)):
        want_y, want_g = prior.get_y(labels, start), prior.get_y(guide, start)
        got = prior.calls[2 * w: 2 * w + 2]
        assert [c[0].shape[0] for c in got] == [3, 1] and [c[1].shape[0] for c in got] == [3, 1]
        assert torch.equal(torch.cat([c[0] for c in got]), want_y)
        assert torch.equal(torch.cat([c[1] for c in got]), want_g)
    # the lyrics follow the window: the two windows read different characters of the guidance lyrics
    assert not torch.equal(prior.calls[0][1][:, -12:], prior.calls[2][1][:, -12:])
    # no guidance_labels: the null labels, windowed the same way
    prior.calls.clear()
    zs = [torch.zeros(N, 0, dtype=torch.long)]
    LevelRun(zs, labels, dict(max_batch_size=4, guidance_scale=2.0), 0, prior, None).run_window(Window(0, 8))
    from jukebox_b200.sample import null_labels
    assert torch.equal(prior.calls[0][1], prior.get_y(null_labels(prior, labels), 0))
    # unguided: no guidance keys reach the prior
    prior.calls.clear()
    zs = [torch.zeros(N, 0, dtype=torch.long)]
    LevelRun(zs, labels, dict(max_batch_size=4), 0, prior, None).run_window(Window(0, 8))
    assert prior.calls[0][1] is None and prior.calls[0][2] is None


def test_level_run_refuses_batches_beyond_one_engine():
    from jukebox_b200.sample import LevelRun
    labels = _labels(_LabelPrior(), [dict(artist="a", genre="b", lyrics="", total_length=64, offset=0)] * 2)
    zs = [torch.zeros(2, 0, dtype=torch.long)]
    for limit, bad in ((16, 17), (8, 9)):
        with pytest.raises(ValueError, match=f"at most {limit} guided items"):
            LevelRun(zs, labels, dict(max_batch_size=bad, guidance_scale=2.0), 0, _LabelPrior(limit=limit), None)
        LevelRun(zs, labels, dict(max_batch_size=limit, guidance_scale=2.0), 0, _LabelPrior(limit=limit), None)
    with pytest.raises(ValueError, match="without a guidance_scale"):
        LevelRun(zs, labels, dict(max_batch_size=2, guidance_labels=labels), 0, _LabelPrior(), None)


def test_regenerate_refuses_guidance():
    from jukebox_b200 import sample
    prior = _LabelPrior()
    zs = [torch.zeros(2, 32, dtype=torch.long)]
    for kw in (dict(guidance_scale=2.0), dict(guidance_labels={})):
        with pytest.raises(ValueError, match="guided"):
            sample.regenerate_level(zs, None, dict(kw, max_batch_size=2), 0, prior, 4, 8, None)
        with pytest.raises(ValueError, match="guided"):
            sample.regenerate(zs, [None], [dict(kw, max_batch_size=2)], [prior], 16, 32, None)


def test_simple_prior_without_labels_refuses_guidance():
    class P:
        labeller = EmptyLabeller()
        x_cond = False
        y_cond = False
    p = P()
    with pytest.raises(ValueError, match="no labels"):
        SimplePrior.null_y(p, None)


# ---- codegen ------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"),
                    reason="needs the CUDA toolkit")
def test_guided_kernel_does_not_spill(tmp_path):
    from jukebox_b200.build import _nvcc
    src = os.path.join(ROOT, "jukebox_b200", "csrc", "sampling.cu")
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
           "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "sampling.o"), "-I", os.path.join(ROOT, "include")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    report, current = {}, None
    for line in out.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            report[current] = tuple(int(v) for v in m.groups())
    found = {k: v for k, v in report.items() if "sample_guided_kernel" in k}
    assert sorted(re.search(r"ILi(\d+)E", k).group(1) for k in found) == ["16", "4", "8"], report
    for name, (stack, st, ld) in found.items():
        assert stack == 0 and st == 0 and ld == 0, f"{name}: {stack} bytes stack, spills {st} / {ld} bytes"
