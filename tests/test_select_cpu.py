"""Sample selection without a GPU: the plan of jk_prior_select (which rows are stashed) simulated on host arrays against a
direct gather for every parent vector of up to 5 rows and random ones of 16 and 32; bad input; the keep-best ranking;
the C ABI of the new symbols; and the host flow of SamplingWindow.select / a one-row prime / LevelRun's ancestry, with
a fake engine."""
import ctypes as C
import itertools
import os
import random
import shutil
import subprocess
import tempfile

import pytest
import torch

import jukebox_b200.prior.autoregressive as ar
from jukebox_b200 import _lib
from jukebox_b200.engine import prior_config, select_plan
from jukebox_b200.prior.autoregressive import keep_best_parents

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# every attn_func, 6 and 7 included: rows per (sample, head) n_ctx, bc, n_ctx, 2 bc, encoder_dims, padded prime
CFG = dict(width=128, depth=6, heads=2, n_state=96, mlp_width=128, n_ctx=64, blocks=8, attn_funcs=[0, 1, 2, 3, 6, 7],
           bins=40, prime_len=10, encoder_dims=12, max_batch=32)


def _row_bytes(c):
    dh_pad = (c["n_state"] // c["heads"] + 15) // 16 * 16
    bc = c["n_ctx"] // c["blocks"]
    rows = {0: c["n_ctx"], 1: bc, 2: c["n_ctx"], 3: 2 * bc, 6: c["encoder_dims"],
            7: (c["prime_len"] // c["blocks"] + 1) * c["blocks"]}
    return sum(2 * c["heads"] * rows[f] * dh_pad * 2 for f in c["attn_funcs"])


def _simulate(parents, info):
    """the two launches of jk_prior_select on labelled rows: stash, then every copy reading the pre-copy state; a copy
    may read a row directly only if no copy of the same launch writes it"""
    n = len(parents)
    rows = list(range(n))
    stash = [rows[s] for s in info.stash[:info.n_stash]]
    slot = {s: i for i, s in enumerate(info.stash[:info.n_stash])}
    dsts = {b for b in range(n) if parents[b] != b}
    out = list(rows)
    for b in sorted(dsts):
        s = parents[b]
        if s in slot:
            out[b] = stash[slot[s]]
        else:
            assert s not in dsts, f"{parents}: row {s} is read directly and overwritten in the same launch"
            out[b] = rows[s]
    return out


def _check(cfg, parents):
    info = select_plan(cfg, parents)
    n = len(parents)
    assert _simulate(parents, info) == [parents[b] for b in range(n)], parents
    read = {parents[b] for b in range(n) if parents[b] != b}
    want_stash = sorted(r for r in read if parents[r] != r)
    assert list(info.stash[:info.n_stash]) == want_stash, parents
    copies = sum(parents[b] != b for b in range(n))
    assert info.n_copies == copies
    rb = _row_bytes(CFG)
    assert info.row_bytes == rb
    assert info.workspace_bytes == rb * len(want_stash)
    assert info.bytes_moved == 2 * rb * (len(want_stash) + copies)
    return info


def test_plan_matches_a_direct_gather_for_every_small_parent_vector():
    cfg = prior_config(**CFG)
    for n in range(1, 6):
        for parents in itertools.product(range(n), repeat=n):
            _check(cfg, list(parents))


@pytest.mark.parametrize("n", [16, 32])
def test_plan_matches_a_direct_gather_for_random_parent_vectors(n):
    cfg = prior_config(**CFG)
    rng = random.Random(n)
    for _ in range(300):
        kind = rng.randrange(3)
        if kind == 0:
            parents = [rng.randrange(n) for _ in range(n)]
        elif kind == 1:
            parents = list(range(n))
            rng.shuffle(parents)
        else:                                        # a permutation of a few rows, the rest in place
            parents = list(range(n))
            sub = rng.sample(range(n), rng.randrange(2, 6))
            for a, b in zip(sub, sub[1:] + sub[:1]):
                parents[a] = b
        _check(cfg, parents)


def test_identity_broadcast_and_keep_best_stash_nothing():
    cfg = prior_config(**CFG)
    for n in (1, 5, 16, 32):
        ident = _check(cfg, list(range(n)))
        assert ident.n_copies == 0 and ident.bytes_moved == 0 and ident.workspace_bytes == 0
        bc = _check(cfg, [0] * n)
        assert bc.n_stash == 0 and bc.n_copies == n - 1
        rng = random.Random(n)
        for keep in range(1, n + 1):
            info = _check(cfg, keep_best_parents([rng.choice([-1.0, -2.0, -3.5]) for _ in range(n)], keep))
            assert info.n_stash == 0 and info.n_copies == n - keep
    # a swap, a 3-cycle and a reversal stash what they overwrite and read
    assert list(_check(cfg, [1, 0, 2, 3]).stash[:2]) == [0, 1]
    assert _check(cfg, [1, 2, 0, 3, 3]).n_stash == 3
    assert _check(cfg, list(range(31, -1, -1))).n_stash == 32


def test_bad_selections_are_rejected_with_a_message():
    cfg = prior_config(**dict(CFG, max_batch=8))
    for parents, msg in (([], "rows"), ([0] * 9, "out of range"), ([0, -1], "outside"), ([0, 2], "outside"),
                         ([0] * 40, "rows")):
        with pytest.raises(RuntimeError, match=msg):
            select_plan(cfg, parents)
    with pytest.raises(RuntimeError, match="attn_func 5"):
        select_plan(prior_config(**dict(CFG, attn_funcs=[0, 1, 2, 3, 6, 5])), [0, 0])
    with pytest.raises(RuntimeError, match="integer"):
        select_plan(cfg, torch.zeros(2))


def test_keep_best_ranking():
    # kept rows keep their slots; the others, ascending, copy the kept rows round-robin in rank order
    assert keep_best_parents([-5.0, -1.0, -3.0, -2.0, -9.0, -4.0], 2) == [1, 1, 3, 3, 1, 3]
    assert keep_best_parents([-5.0, -1.0, -3.0, -2.0, -9.0, -4.0], 3) == [1, 1, 2, 3, 3, 2]
    # ties go to the lower row, nan ranks last
    assert keep_best_parents([-1.0, -1.0, -1.0, -1.0], 1) == [0, 0, 0, 0]
    assert keep_best_parents([-2.0, -1.0, -1.0, -2.0], 2) == [1, 1, 2, 2]
    assert keep_best_parents([float("nan"), -7.0, -8.0], 1) == [1, 1, 1]
    assert keep_best_parents([-3.0, -2.0, -1.0], 3) == [0, 1, 2]
    with pytest.raises(AssertionError):
        keep_best_parents([0.0, 1.0], 3)


def test_select_symbols_and_struct_match_the_header():
    assert _lib.SIGNATURES["jk_prior_select_plan"] == (
        C.c_int, [C.POINTER(_lib.PriorConfig), C.POINTER(C.c_int32), C.c_int, C.POINTER(_lib.SelectPlanInfo)])
    assert _lib.SIGNATURES["jk_prior_select"] == (
        C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p])
    lib = _lib.lib()
    for name in ("jk_prior_select_plan", "jk_prior_select"):
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    if shutil.which("gcc") is None:
        pytest.skip("needs gcc for the struct layout")
    fields = [f[0] for f in _lib.SelectPlanInfo._fields_]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "jkb200.h"', "int main(void) {",
            'printf("%zu\\n", sizeof(jk_select_plan_info));']
    prog += ['printf("%%zu\\n", offsetof(jk_select_plan_info, %s));' % f for f in fields]
    prog += ["return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "abi.c"), os.path.join(d, "abi")
        open(src, "w").write("\n".join(prog))
        subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        vals = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert vals[0] == C.sizeof(_lib.SelectPlanInfo)
    assert vals[1:] == [getattr(_lib.SelectPlanInfo, f).offset for f in fields]


# ---- host flow with a fake engine ---------------------------------------------------------------------------------
class FakeEngine:
    """rows carry a label: the row they were first prefilled / stepped as, permuted by select"""

    def __init__(self, capacity, N):
        self.prefill_capacity = capacity
        self.has_logits_gemm = False
        self.calls = []
        self.position = 0
        self.rows = list(range(N))

    def reset(self, t0=0):
        self.position = t0

    def set_encoder_kv(self, enc):
        self.calls.append(("enc", enc.shape[0]))

    def prefill(self, n, P, **kw):
        self.calls.append(("prefill", n, P))
        self.position = P

    def step(self, n, tokens=None, logits=None, **kw):
        self.calls.append(("step", n, self.position))
        if logits is not None:
            logits.zero_()
        self.position += 1

    def select(self, parents):
        self.calls.append(("select", list(parents)))
        self.rows = [self.rows[p] for p in parents]


def _model(monkeypatch, capacity, N, score):
    m = ar.ConditionalAutoregressive2D((24,), 16, width=64, depth=2, heads=1, attn_order=0, blocks=None).eval()
    eng = FakeEngine(capacity, N)
    monkeypatch.setattr(m, "_engine", lambda n: eng)
    monkeypatch.setattr(m.transformer, "check_cache", lambda *a, **k: None)

    def fake_scored(logits, raw, temp, seed, position, tokens, logp):
        n = tokens.shape[0]
        assert logp.shape[0] == n == raw.shape[0]
        if logits is not None:                       # a row draws its engine label; its score follows the label too
            tokens[:, position] = torch.tensor(eng.rows[:n]) + 1
        logp[:, position] = torch.tensor([score(r, position) for r in eng.rows[:n]])
    monkeypatch.setattr(ar, "sample_categorical_scored", fake_scored)
    monkeypatch.setattr(ar, "sample_categorical", lambda *a: pytest.fail("selection scores every draw"))
    import jukebox_b200.score as score_mod
    monkeypatch.setattr(score_mod, "xout_logprob", lambda h, w, targets: torch.full((h.shape[0],), -1.0))
    return m, eng


def test_keep_best_window_reorders_every_row_tensor(monkeypatch):
    N, k, keep = 4, 2, 3
    m, eng = _model(monkeypatch, 512, N, lambda r, t: -float(r))           # a row drawn as label r scores -r
    prime = torch.arange(N * 3).view(N, 3) % 16
    z, lp, anc = m.primed_sample(N, prime, fp16=True, sample_tokens=7, get_logprobs=True, select_every=k,
                                 select_keep=keep)
    sels = [c[1] for c in eng.calls if c[0] == "select"]
    # drawn tokens 3, 4: scores 0, -2, -4, -6 -> rows 0, 1, 2 kept, row 3 copies row 0.  Drawn 5, 6 (the last): scores
    # 0, -4, -8 and 0 inherited from row 0 -> ranks 0, 3, 1 kept (tie to the lower row), row 2 copies row 0
    assert sels == [[0, 1, 2, 0], [0, 1, 0, 3]]
    assert anc.tolist() == [0, 1, 0, 0]
    assert torch.equal(z[:, :3], prime[anc])                                # the given tokens follow their item
    assert z[:, 3:].tolist() == [[1] * 4, [2] * 4, [1] * 4, [1] * 4]
    assert lp[:, 3:].tolist() == [[0.0] * 4, [-1.0] * 4, [0.0] * 4, [0.0] * 4]
    # selection off: the same call without it returns no ancestry and never selects
    eng.calls.clear()
    eng.rows = list(range(N))
    out = m.primed_sample(N, prime, fp16=True, sample_tokens=7, get_logprobs=True)
    assert len(out) == 2 and not [c for c in eng.calls if c[0] == "select"]


def test_selection_options_are_checked(monkeypatch):
    m, eng = _model(monkeypatch, 512, 4, lambda r, t: 0.0)
    for kw in (dict(select_every=2), dict(select_keep=2), dict(select_every=0, select_keep=1),
               dict(select_every=2, select_keep=5)):
        with pytest.raises(ValueError):
            m.sample(4, fp16=True, sample_tokens=4, **kw)


@pytest.mark.parametrize("capacity", [512, 0])
def test_one_row_prime_runs_once_then_every_row_continues_it(monkeypatch, capacity):
    N = 3
    m, eng = _model(monkeypatch, capacity, N, lambda r, t: -1.0)
    prime = torch.tensor([[3, 4, 5, 6]])
    z, lp = m.primed_sample(N, prime, fp16=True, sample_tokens=6, get_logprobs=True)
    given = [c for c in eng.calls if c[0] in ("prefill", "step") and (c[1] == 1)]
    if capacity:
        assert eng.calls[0] == ("prefill", 1, 4)
    else:
        assert given == [("step", 1, t) for t in range(4)]
    i = eng.calls.index(("select", [0] * N))
    assert all(c[1] == N for c in eng.calls[i + 1:] if c[0] == "step")
    assert [c[2] for c in eng.calls[i + 1:]] == [4, 5]
    assert torch.equal(z[:, :4], prime.repeat(N, 1)) and z.shape == (N, 6)
    assert lp.shape == (N, 6) and bool((lp == -1.0).all())


def test_level_run_moves_every_level_with_its_item():
    from jukebox_b200.sample import LevelRun, Window

    class FakePrior:
        n_ctx, level = 8, 0

        def get_z_conds(self, zs, start, end):
            return [zs[1][:, start // 2:end // 2]]

        def get_y(self, labels, start):
            return labels["y"]

        def sample(self, n_samples, z, z_conds, y, **kw):
            assert kw["select_every"] == 2
            anc = torch.arange(n_samples).flip(0)
            new = torch.full((n_samples, self.n_ctx - z.shape[1]), 7)
            return torch.cat([z[anc], new], 1), anc

    N = 4
    zs = [torch.arange(N).view(N, 1).repeat(1, 3), torch.arange(N).view(N, 1).repeat(1, 4) + 10]
    labels = dict(y=torch.zeros(N, 5, dtype=torch.long))
    run = LevelRun(zs, labels, dict(max_batch_size=2, select_every=2, select_keep=1), 0, FakePrior(), None)
    run.run_window(Window(0, 8))
    # pieces of 2 rows: each piece reversed within itself, at both levels
    assert zs[0][:, 0].tolist() == [1, 0, 3, 2] and zs[0].shape == (N, 8)
    assert zs[1][:, 0].tolist() == [11, 10, 13, 12]
    zs = [zs[0][:, :3], zs[1]]
    labels["y"][3, 1] = 1
    with pytest.raises(ValueError, match="different labels"):
        LevelRun(zs, labels, dict(max_batch_size=2, select_every=2, select_keep=1), 0, FakePrior(), None).run_window(
            Window(0, 8))
