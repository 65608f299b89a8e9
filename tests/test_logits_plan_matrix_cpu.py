"""The logits plans that tests/test_gpu_logits_exact.py runs, pinned on the host (jk_prior_plan at 132 SMs, the H100 SXM;
no GPU).  The engine computes the logits by the tensor-core GEMM in 1 to 4 passes or by the fp32 FMA product; which one
depends on the K split, the vocabulary, the row layout and two environment switches.  Each case below is a one-layer
stack at a released model's width and vocabulary (or a vocabulary chosen to reach a pass count), and this file checks
that the matrix as a whole reaches every route, so the GPU file's coverage holds even where it cannot check it itself."""
import ctypes as C
from collections import namedtuple

import pytest

from jukebox_b200 import _lib

N_CTX = 64      # context of the test engines: the logits do not depend on it

# runs: (max_batch the engine is planned for, samples stepped); plans: max_batch -> (k_split, logits_passes) at 132 SMs
Case = namedtuple("Case", "width heads bins env runs plans")
_1B = dict(width=2048, heads=2, bins=2127)
CASES = {
    # the production plan: ragged vocabulary, two passes, every row layout, and an engine planned for 32 stepped at 16 and
    # 9 samples (the 16-row kernel on the 32-row layout)
    "1b_lyrics": Case(**_1B, env={}, runs=[(1, 1), (8, 8), (16, 16), (17, 17), (32, 32), (32, 16), (32, 9)],
                      plans={mb: (4, 2) for mb in (1, 8, 16, 17, 32)}),
    "small_upsampler": Case(1024, 1, 1024, {}, [(16, 16), (32, 32)], {16: (4, 1), 32: (4, 1)}),
    # [32 x (2 * 1920 / 2 + 8)] fp16 GEMM tile does not fit at 32 rows: the FMA logits at R = 32
    "upsampler_level_0": Case(1920, 1, 2048, {}, [(16, 16), (32, 32)], {16: (2, 1), 32: (2, 0)}),
    # n_state 288 is 18 k-steps, which do not split 4 ways: K split 2, and its tile fits at 32 rows
    "ksplit2_rows32": Case(1152, 2, 4500, {}, [(16, 16), (32, 32)], {16: (2, 2), 32: (2, 2)}),
    # K split 1 (600 groups of the 4800-wide Conv1Ds over 33 or 66 units exceed 8 per unit): FMA logits, and the K tile of
    # 1024 floats does not divide 4800
    "5b_lyrics": Case(4800, 8, 2048, {}, [(1, 1), (8, 8), (16, 16)], {1: (1, 0), 8: (1, 0), 16: (1, 0)}),
    "passes3": Case(1024, 1, 4500, {}, [(16, 16), (32, 32)], {16: (4, 3), 32: (4, 3)}),        # 563 groups, ragged
    "passes4": Case(1024, 1, 8448, {}, [(16, 16), (32, 32)], {16: (4, 4), 32: (4, 4)}),        # 1056 = 33 x 32 groups
    "passes5": Case(1024, 1, 8449, {}, [(16, 16)], {16: (4, 0)}),                              # 33 groups on a unit
    # [16 x (4096 / 2 + 8)] fp16 is 65 792 bytes, 256 over the 64 KB the union region holds at 16 rows
    "1b_ksplit2": Case(**_1B, env={"JK_KSPLIT": "2"}, runs=[(16, 16)], plans={16: (2, 0)}),
    "1b_ksplit1": Case(**_1B, env={"JK_KSPLIT": "1"}, runs=[(16, 16), (32, 32)], plans={16: (1, 0), 32: (1, 0)}),
    "1b_no_logits_mma": Case(**_1B, env={"JK_NO_LOGITS_MMA": "1"}, runs=[(16, 16), (32, 32)],
                             plans={16: (4, 0), 32: (4, 0)}),
}


def layout_rows(max_batch):
    """rows of the engine's shared-memory layout: the 32-row kernel's above 16 samples, an 8-row A tile up to 8"""
    return 32 if max_batch > 16 else 16 if max_batch > 8 else 8


def prior_config(case, max_batch):
    cfg = _lib.PriorConfig()
    cfg.width, cfg.depth, cfg.heads, cfg.n_state, cfg.mlp_width = case.width, 1, case.heads, case.width // 4, case.width
    cfg.n_ctx, cfg.blocks, cfg.bins, cfg.prime_len, cfg.encoder_dims = N_CTX, 0, case.bins, 0, 0
    cfg.max_batch, cfg.add_cond_after = max_batch, 1
    cfg.attn_func[0] = 0
    return cfg


def plan_info(case, max_batch, sms):
    """jk_prior_plan of the case (the caller sets the case's environment first: the planner reads it)"""
    info = _lib.PlanInfo()
    _lib.check(_lib.lib().jk_prior_plan(C.byref(prior_config(case, max_batch)), sms, C.byref(info), None, 0))
    return info


def set_case_env(monkeypatch, case):
    for k in ("JK_KSPLIT", "JK_NO_LOGITS_MMA"):
        monkeypatch.delenv(k, raising=False)
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("name", list(CASES))
def test_case_plan_at_132_sms(name, monkeypatch):
    case = CASES[name]
    set_case_env(monkeypatch, case)
    assert sorted(case.plans) == sorted({mb for mb, _ in case.runs})
    for mb, n in case.runs:
        assert 1 <= n <= mb
    for mb, want in case.plans.items():
        info = plan_info(case, mb, 132)
        assert (info.k_split, info.logits_passes) == want, (name, mb, info.k_split, info.logits_passes)
        assert info.units * info.k_split == 132


def test_5b_lyrics_plan_has_three_ring_slots_at_16_samples(monkeypatch):
    set_case_env(monkeypatch, CASES["5b_lyrics"])
    assert plan_info(CASES["5b_lyrics"], 16, 132).ring_slots == 3


def test_passes5_needs_more_than_four_passes():
    # the pass limit, not the tile or the K split, turns the GEMM off: one more column than passes4
    for name, passes in (("passes4", 4), ("passes5", 5)):
        case = CASES[name]
        units = 132 // case.plans[16][0]
        groups = (case.bins + 7) // 8
        assert (-(-groups // units) + 7) // 8 == passes


def test_matrix_reaches_every_logits_route():
    plans = [(CASES[name], mb, ks, np_) for name in CASES for mb, (ks, np_) in CASES[name].plans.items()]
    gemm = [(c, mb, ks, np_) for c, mb, ks, np_ in plans if np_ > 0]
    fma = [(c, mb, ks, np_) for c, mb, ks, np_ in plans if np_ == 0]
    assert {np_ for _, _, _, np_ in gemm} == {1, 2, 3, 4}
    assert {ks for _, _, ks, _ in plans} == {1, 2, 4}
    # K split 2 runs the GEMM at both row counts
    assert {layout_rows(mb) for _, mb, ks, _ in gemm if ks == 2} == {16, 32}
    assert {layout_rows(mb) for _, mb, _, _ in gemm} == {8, 16, 32}
    # the FMA fallback at 32 rows of a configuration whose 16-row plan has the GEMM, with no switch set
    assert any(layout_rows(mb) == 32 and not c.env and c.plans[16][1] > 0 for c, mb, _, _ in fma)
    # both the 16- and 32-row kernels step an engine whose layout has 32 rows
    assert {n for c in CASES.values() for mb, n in c.runs if layout_rows(mb) == 32 and n <= 16}
    # odd vocabularies (a padded last column in the GEMM's last pair) with the GEMM
    assert any(c.bins % 2 for c, _, _, _ in gemm)
