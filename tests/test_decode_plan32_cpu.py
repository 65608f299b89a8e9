"""Host-side planning of the decode engine at 32 samples (jk_prior_plan, no GPU): more than 16 samples take the 32-row
kernel, whose shared-memory layout differs, while the K split, the column ownership and the logits passes stay those of
the 16-row plan."""
import ctypes as C

import numpy as np
import pytest

from jukebox_b200 import _lib
from test_decode_plan_cpu import CONFIGS
from jukebox_b200.transformer.transformer import attn_func_of


def plan(name, max_batch, sms=132):
    w, depth, heads, n_ctx, blocks, order, prime, enc, bins, _, _ = CONFIGS[name]
    cfg = _lib.PriorConfig()
    cfg.width, cfg.depth, cfg.heads, cfg.n_state, cfg.mlp_width = w, depth, heads, w // 4, w
    cfg.n_ctx, cfg.blocks, cfg.bins, cfg.prime_len, cfg.encoder_dims = n_ctx, blocks, bins, prime, enc
    cfg.max_batch, cfg.add_cond_after = max_batch, 1
    for d in range(depth):
        cfg.attn_func[d] = attn_func_of(order, d)
    info = _lib.PlanInfo()
    cols = (C.c_uint16 * (sms * depth * 4 * 2 + 8 * sms))()
    rc = _lib.lib().jk_prior_plan(C.byref(cfg), sms, C.byref(info), cols, len(cols))
    return rc, info, np.frombuffer(cols, dtype=np.uint16).copy()


@pytest.mark.parametrize("name", ["1b_lyrics", "small_upsampler", "upsampler_level_0", "5b_lyric_encoder"])
def test_plan_at_32_samples(name):
    rc16, info16, cols16 = plan(name, 16)
    rc, info, cols = plan(name, 32)
    assert rc16 == 0 and rc == 0, _lib.lib().jk_last_error()
    assert info.k_split == info16.k_split == CONFIGS[name][-1] and info.units == info16.units
    n = info.units * CONFIGS[name][1] * 4 * 2
    assert (cols[:n] == cols16[:n]).all()                       # same column table of every layer
    assert info.smem_bytes <= 232448
    assert info.ring_slots >= 4
    if name == "upsampler_level_0":
        # its [32 x (2 * 1920 / 2 + 8)] logits GEMM tile (123 KB) does not fit: the fp32 FMA logits run instead
        assert info16.logits_passes == 1 and info.logits_passes == 0
    else:
        assert info.logits_passes == info16.logits_passes
        assert (cols == cols16).all() and info.stream_stride == info16.stream_stride
    assert info.arena_bytes > info16.arena_bytes                # KV caches for twice the samples
    print(name, dict(ring_slots=(info16.ring_slots, info.ring_slots), tile_rows=(info16.tile_rows, info.tile_rows),
                     smem=(info16.smem_bytes, info.smem_bytes), arena_gb=info.arena_bytes / 1e9))


def test_1b_lyrics_keeps_the_logits_gemm_at_32():
    _, info, _ = plan("1b_lyrics", 32)
    assert info.logits_passes == 2


def test_more_than_16_rejected_where_the_32_row_tile_cannot_fit():
    rc, _, _ = plan("5b_lyrics", 32)                            # K split 1: a [32 x 4808] fp16 tile is 308 KB
    assert rc != 0
    msg = _lib.lib().jk_last_error()
    assert b"232448" in msg and b"at most 16 samples" in msg, msg
    assert plan("5b_lyrics", 16)[0] == 0


@pytest.mark.parametrize("name", list(CONFIGS))
def test_33_samples_rejected(name):
    rc, _, _ = plan(name, 33)
    assert rc != 0
    assert b"max_batch 33 out of range (<= 32)" in _lib.lib().jk_last_error()


def test_16_sample_plan_unchanged_by_the_32_row_kernel():
    # an engine planned for <= 16 samples keeps the 16-row layout it had before the 32-row kernel existed
    for name, slots, smem in (("1b_lyrics", 6, 221184), ("upsampler_level_0", 7, 219136)):
        _, info, _ = plan(name, 16)
        assert (info.ring_slots, info.smem_bytes) == (slots, smem), (name, info.ring_slots, info.smem_bytes)
