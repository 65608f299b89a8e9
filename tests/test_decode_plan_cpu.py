"""Host-side planning of the decode engine (jk_prior_plan: pure arithmetic, no GPU): K-split units, column ownership,
shared-memory budget - for the BASELINE configurations on a 132-SM device (H100 SXM)."""
import ctypes as C

import numpy as np
import pytest

from jukebox_b200 import _lib
from jukebox_b200.transformer.transformer import attn_func_of

CONFIGS = {
    # name: (width, depth, heads, n_ctx, blocks, attn_order, prime_len, encoder_dims, bins, max_batch, expected k_split)
    "1b_lyrics": (2048, 72, 2, 8576, 64, 12, 384, 0, 2127, 16, 4),
    "5b_lyrics": (4800, 79, 8, 8192, 128, 10, 0, 512, 2048, 8, 1),
    "5b_lyric_encoder": (1280, 18, 4, 512, 32, 2, 0, 0, 0, 8, 4),
    "small_upsampler": (1024, 48, 1, 8192, 64, 2, 0, 0, 1024, 16, 4),
    "upsampler_level_0": (1920, 72, 1, 8192, 128, 2, 0, 0, 2048, 16, 2),
    "tiny": (64, 8, 2, 48, 4, 9, 0, 0, 50, 3, 1),
}


def plan(name, sms=132):
    w, depth, heads, n_ctx, blocks, order, prime, enc, bins, mb, _ = CONFIGS[name]
    cfg = _lib.PriorConfig()
    cfg.width, cfg.depth, cfg.heads, cfg.n_state, cfg.mlp_width = w, depth, heads, w // 4, w
    cfg.n_ctx, cfg.blocks, cfg.bins, cfg.prime_len, cfg.encoder_dims = n_ctx, blocks, bins, prime, enc
    cfg.max_batch, cfg.add_cond_after = mb, 1
    for d in range(depth):
        cfg.attn_func[d] = attn_func_of(order, d)
    info = _lib.PlanInfo()
    cols = (C.c_uint16 * (sms * depth * 4 * 2))()
    _lib.check(_lib.lib().jk_prior_plan(C.byref(cfg), sms, C.byref(info), cols, len(cols)))
    units = info.units
    arr = np.frombuffer(cols, dtype=np.uint16)[: units * depth * 8].reshape(units, depth, 4, 2).astype(np.int64)
    return cfg, info, arr


@pytest.mark.parametrize("name", list(CONFIGS))
def test_units_partition_every_conv1d(name):
    cfg, info, cols = plan(name)
    assert info.k_split == CONFIGS[name][-1]
    assert info.units * info.k_split == 132
    assert 2 <= info.ring_slots <= 12 and info.smem_bytes <= 232448
    S, W, M = cfg.n_state, cfg.width, cfg.mlp_width
    for l in range(cfg.depth):
        n_out = [S if cfg.attn_func[l] == 6 else 3 * S, W, M, W]
        for gi in range(4):
            g0, ncg = cols[:, l, gi, 0], cols[:, l, gi, 1]
            assert (ncg <= 8).all()
            assert int(ncg.sum()) == n_out[gi] // 8                       # every 8-column group owned exactly once ...
            assert (g0 == np.concatenate([[0], np.cumsum(ncg)[:-1]])).all()   # ... contiguously, in unit order
            assert ((ncg * 4) % info.k_split == 0).all()                   # column pairs split evenly over the unit's CTAs
    # the residual stream stays in the shared memory of the CTA that finishes it: proj and proj2 columns never move
    assert (cols[:, :, 1] == cols[:, :1, 1]).all() and (cols[:, :, 3] == cols[:, :1, 1]).all()
    for k_dim in (W, S, M):
        assert (k_dim // 16) % info.k_split == 0


def test_weight_streams_are_balanced():
    cfg, info, cols = plan("1b_lyrics")
    k = np.array([cfg.width, cfg.n_state, cfg.width, cfg.mlp_width]) // info.k_split
    per_unit = (cols[:, :, :, 1] * (k // 16)[None, None, :] * 256).sum((1, 2))
    assert per_unit.max() <= info.stream_stride
    assert per_unit.max() / per_unit.min() < 1.03, (per_unit.min(), per_unit.max())
    total = per_unit.sum() * info.k_split
    assert abs(total - 72 * 12.58e6 * 2) / total < 0.01          # 1.81 GB of fp16 weights, each byte in exactly one stream


def test_plan_rejects_bad_geometry():
    cfg, _, _ = plan("tiny")
    cfg.n_state = 24                                             # not a multiple of 16
    info = _lib.PlanInfo()
    assert _lib.lib().jk_prior_plan(C.byref(cfg), 132, C.byref(info), None, 0) != 0
    assert b"multiples of 16" in _lib.lib().jk_last_error()
