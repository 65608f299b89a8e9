"""The chunked prefill's kernel entry points without a GPU: the float64 reference's key masks and exact-grid inputs of
test_gpu_prefill_attn.py, and every argument jk_prefill_attention_f16 and jk_prefill_gemm_f16 refuse.  The refusals are
checked with fake device addresses: each check runs before any CUDA call, so a call that got past them would fail on a
machine without a GPU with a CUDA error instead of the message asserted here."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

from oracle.attn_layout_np import reference_keys
from test_gpu_prefill_attn import exact_grid, key_lists, key_mask

BASE = 0x7f0000000000                 # fake, 256-byte aligned device addresses; nothing is dereferenced


# ---- the reference's masks ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,bc,prime", [(1, 16, 48), (61, 16, 48), (200, 65, 1), (130, 128, 130), (300, 7, 299)])
@pytest.mark.parametrize("attn_func", [0, 1, 2, 3, 7])
def test_key_masks_are_the_reference_patterns(attn_func, P, bc, prime):
    mask = key_mask(attn_func, P, bc, prime)
    idx, valid = key_lists(mask)
    for p in range(P):
        want = reference_keys(attn_func, p, bc, prime)
        assert mask[p].nonzero().flatten().tolist() == want, (attn_func, p)
        assert idx[p][valid[p]].tolist() == want, (attn_func, p)


def test_encoder_decoder_mask_is_every_row():
    mask = key_mask(6, 5, 0, 0, enc_rows=33)
    assert mask.shape == (5, 33) and bool(mask.all())


# ---- exact-grid inputs ----------------------------------------------------------------------------------------------------
def test_exact_grid_dots_are_exact_in_float32_in_any_order():
    """q with rows up to the widest range the GPU tests draw (24) and k in [-8, 8], over the longest head (480): the dot
    products in float32 under shuffled summation orders are bitwise the float64 ones"""
    g = torch.Generator().manual_seed(3)
    dh = 480
    q = exact_grid((64, dh), torch.randint(1, 25, (64, 1), generator=g), g)
    k = exact_grid((96, dh), 8, g)
    assert q.abs().max() <= 6 and k.abs().max() <= 2
    assert torch.equal(q.float().half(), q)
    want = q.double() @ k.double().t()
    prods = q.float()[:, None, :] * k.float()[None, :, :]                # exact: multiples of 2^-4
    for trial in range(4):
        perm = torch.randperm(dh, generator=g)
        acc = torch.zeros(64, 96, dtype=torch.float32)
        for d in perm.tolist():
            acc += prods[..., d]
        assert torch.equal(acc.double(), want), trial
        assert torch.equal(prods[..., perm].sum(-1).double(), want), trial    # torch's own (blocked) order


# ---- attention refusals -----------------------------------------------------------------------------------------------
def _attn_args(**kw):
    from jukebox_b200 import _lib
    a = dict(qkv=BASE, k_cache=None, v_cache=None, out=BASE + 0x1000000, w=None, ld=0, n=2, P=100, heads=2, dh=64,
             dh_pad=64, attn_func=0, bc=0, prime=0, enc_rows=0, route=0)
    a.update(kw)
    return _lib.PrefillAttnArgs(**a)


def _attn_call(**kw):
    from jukebox_b200._lib import PrefillAttnRoute, lib
    taken = PrefillAttnRoute(7, 7, 7)
    rc = lib().jk_prefill_attention_f16(C.byref(_attn_args(**kw)), C.byref(taken), None)
    assert (taken.tensor_cores, taken.tile_dh, taken.stage_bytes) == (7, 7, 7), "a refused call reported a route"
    return rc, lib().jk_last_error().decode()


ENC = dict(attn_func=6, enc_rows=33, k_cache=BASE + 0x2000000, v_cache=BASE + 0x3000000)
ATTN_REFUSALS = [
    (dict(attn_func=4), "attn_func 4"),
    (dict(attn_func=5), "attn_func 5"),
    (dict(attn_func=8), "attn_func 8"),
    (dict(attn_func=-1), "attn_func -1"),
    (dict(dh=80, dh_pad=64), "dh_pad 64"),
    (dict(dh=40, dh_pad=40), "dh_pad 40"),
    (dict(dh=150, dh_pad=152), "dh_pad 152"),
    (dict(attn_func=1, bc=0), "bc >= 1"),
    (dict(attn_func=2, bc=0), "bc >= 1"),
    (dict(attn_func=3, bc=-4), "bc >= 1"),
    (dict(attn_func=7, prime=0), "prime >= 1"),
    (dict(ENC, enc_rows=0), "enc_rows >= 1"),
    (dict(ENC, k_cache=None), "both caches"),
    (dict(ENC, v_cache=None), "both caches"),
    (dict(w=BASE + 0x4000000, ld=0), "ld >= 1"),
    (dict(out=None, w=BASE + 0x4000000, ld=-1), "ld >= 1"),
    (dict(out=None), "neither out nor w"),
    (dict(qkv=BASE + 8), "16-byte aligned"),
    (dict(qkv=BASE + 2), "16-byte aligned"),
    (dict(out=BASE + 0x1000004), "16-byte aligned"),
    (dict(ENC, k_cache=BASE + 0x2000008), "16-byte aligned"),
    (dict(ENC, v_cache=BASE + 0x3000002), "16-byte aligned"),
    (dict(route=2), "route 2"),
    (dict(n=0), "empty shape"),
    (dict(P=0), "empty shape"),
    # the scalar kernels keep q and one score per key in 64 KB of shared memory
    (dict(dh=480, dh_pad=480, P=16000), "shared memory"),
    (dict(dh=75, dh_pad=80, P=16310), "shared memory"),
    (dict(route=1, P=16321), "shared memory"),
    (dict(ENC, route=1, enc_rows=20000, P=10), "shared memory"),
]


@pytest.mark.parametrize("kw,msg", ATTN_REFUSALS, ids=[m + "-" + "-".join(f"{k}{v}" for k, v in kw.items() if k in
                                                                         ("attn_func", "dh", "P", "route", "ld"))
                                                       for kw, m in ATTN_REFUSALS])
def test_prefill_attention_refuses_before_any_launch(kw, msg):
    rc, err = _attn_call(**kw)
    assert rc != 0
    assert msg in err, err


def test_prefill_attention_scalar_limit_is_exact():
    """(dh + max(P, enc_rows)) * 4 <= 64 KB: one float over is refused, the limit itself passes the checks (and then
    fails on the missing device, not on the limit)"""
    rc, err = _attn_call(dh=75, dh_pad=80, P=16384 - 75 + 1)
    assert rc != 0 and "shared memory" in err
    if not torch.cuda.is_available():
        rc, err = _attn_call(dh=75, dh_pad=80, P=16384 - 75)
        assert rc != 0 and "shared memory" not in err, err


# ---- GEMM refusals --------------------------------------------------------------------------------------------------
def _gemm_call(x=BASE, w_t=BASE + 0x1000000, res=None, y=BASE + 0x2000000, M=128, N=128, K=128, epi=0):
    from jukebox_b200._lib import lib
    rc = lib().jk_prefill_gemm_f16(x, w_t, None, res, y, M, N, K, epi, None)
    return rc, lib().jk_last_error().decode()


GEMM_REFUSALS = [
    (dict(K=56), "K >= 64"),
    (dict(K=0), "K >= 64"),
    (dict(K=68), "K % 8 == 0"),
    (dict(K=4801), "K % 8 == 0"),
    (dict(M=0), "K >= 64"),
    (dict(N=0), "K >= 64"),
    (dict(x=BASE + 8), "16-byte aligned"),
    (dict(w_t=BASE + 0x1000002), "16-byte aligned"),
    (dict(y=BASE + 0x2000004), "16-byte aligned"),
    (dict(res=BASE + 0x3000008, epi=2), "16-byte aligned"),
    (dict(epi=2), "bad epilogue 2"),
    (dict(epi=3), "bad epilogue 3"),
    (dict(epi=-1), "bad epilogue -1"),
    (dict(x=None), "null argument"),
    (dict(y=None), "null argument"),
]


@pytest.mark.parametrize("kw,msg", GEMM_REFUSALS, ids=[m + "-" + "-".join(f"{k}{v}" for k, v in kw.items())
                                                       for kw, m in GEMM_REFUSALS])
def test_prefill_gemm_refuses_before_any_launch(kw, msg):
    rc, err = _gemm_call(**kw)
    assert rc != 0
    assert msg in err, err


# ---- the ctypes mirrors ---------------------------------------------------------------------------------------------
def _declared_arity(header, name):
    m = re.search(r"\bint\s+%s\s*\(([^)]*)\)" % name, header, re.S)
    return len([p for p in m.group(1).split(",") if p.strip()])


@pytest.mark.parametrize("name", ["jk_prefill_attention_f16", "jk_prefill_gemm_f16", "jk_conv1d_prefill_f16"])
def test_signatures_match_the_header(name):
    import os
    from jukebox_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "jkb200.h")).read()
    res, args = _lib.SIGNATURES[name]
    assert res is C.c_int and len(args) == _declared_arity(header, name)
    if name == "jk_prefill_attention_f16":
        assert args[0]._type_ is _lib.PrefillAttnArgs and args[1]._type_ is _lib.PrefillAttnRoute
    else:
        assert args[-1] is C.c_void_p and np.all([a in (C.c_void_p, C.c_int) for a in args])
