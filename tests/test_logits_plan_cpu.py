"""Host-side planning of the tensor-core logits GEMM (jk_prior_plan, no GPU): a vocabulary wider than 8 column groups per
unit runs in several passes, each unit multiplying at most 8 groups per pass."""
import ctypes as C

import numpy as np
import pytest

from jukebox_b200 import _lib
from test_decode_plan_cpu import plan


def logits_plan(name, sms):
    cfg, info, layer_cols = plan(name, sms)
    n = info.units * cfg.depth * 4 + info.logits_passes * info.units
    cols = (C.c_uint16 * (2 * n))()
    _lib.check(_lib.lib().jk_prior_plan(C.byref(cfg), sms, C.byref(info), cols, len(cols)))
    arr = np.frombuffer(cols, dtype=np.uint16).astype(np.int64)
    lg = arr[2 * info.units * cfg.depth * 4:].reshape(info.logits_passes, info.units, 2)
    return cfg, info, layer_cols, lg


@pytest.mark.parametrize("sms, passes", [(132, 2), (128, 2), (264, 1)])
def test_1b_lyrics_logits_passes(sms, passes):
    cfg, info, layer_cols, lg = logits_plan("1b_lyrics", sms)
    assert info.logits_passes == passes
    groups = (cfg.bins + 7) // 8
    g0, ncg = lg[:, :, 0], lg[:, :, 1]
    assert (ncg <= 8).all() and ((ncg * 4) % info.k_split == 0).all()
    assert int(ncg.sum()) == groups                                      # every 8-column group of the vocabulary once ...
    total = ncg.sum(0)
    start = np.concatenate([[0], np.cumsum(total)[:-1]])
    assert (g0[0] == start).all()                                        # ... a contiguous range per unit, in unit order,
    for p in range(1, passes):                                           # continued pass after pass
        on = ncg[p] > 0
        assert (g0[p][on] == g0[p - 1][on] + 8).all() and (ncg[p - 1][on] == 8).all()
    assert total.max() - total.min() <= 1
    # the logits streams follow the layers' in every CTA's stream (hi and lo halves: K' = 2 * width)
    k = np.array([cfg.width, cfg.n_state, cfg.width, cfg.mlp_width]) // info.k_split
    per_unit = (layer_cols[:, :, :, 1] * (k // 16)[None, None, :] * 256).sum((1, 2)) + total * (2 * cfg.width // info.k_split // 16) * 256
    assert per_unit.max() <= info.stream_stride


def test_logits_gemm_off_where_it_cannot_run():
    assert logits_plan("5b_lyrics", 132)[1].logits_passes == 0           # K-split 1: the hi / lo halves need two ranks
    assert logits_plan("5b_lyric_encoder", 132)[1].logits_passes == 0    # no vocabulary
    assert logits_plan("small_upsampler", 132)[1].logits_passes == 1     # 128 groups over 33 units
