"""Pointer checks of the residual-block entry points, without a GPU: jk_resblock_cl and jk_resblock_tc are called with
fake device addresses that the kernels could not read with their vector loads.  Both must refuse before any launch:
jk_resblock_cl sends such pointers to its two-launch path, which needs `tmp` (NULL here), and jk_resblock_tc returns an
error naming the alignment it needs."""
import ctypes as C

import pytest

BASE = 0x7f0000000000          # fake, 256-byte aligned device addresses; nothing is dereferenced
NAMES = ("x", "out", "w1", "b1", "w2", "b2")


def _ptrs(misaligned, by):
    return {name: BASE + (i + 1) * 0x100000 + (by if name == misaligned else 0) for i, name in enumerate(NAMES)}


def _call_cl(p, C_, Cs):
    from jukebox_b200._lib import lib
    return lib().jk_resblock_cl(p["x"], p["out"], None, p["w1"], p["b1"], p["w2"], p["b2"], 2, 300, C_, Cs, 3, 0.7, None)


def _call_tc(p, C_, T):
    from jukebox_b200._lib import lib
    return lib().jk_resblock_tc(p["x"], p["out"], p["w1"], p["b1"], p["w2"], p["b2"], 2, T, C_, 3, 0.7, None)


def _error():
    from jukebox_b200._lib import lib
    return lib().jk_last_error().decode()


@pytest.mark.parametrize("C_", [32, 64])
@pytest.mark.parametrize("misaligned,by", [(name, by) for name in NAMES for by in (4, 8)])
def test_resblock_cl_sends_misaligned_pointers_to_the_two_launch_path(misaligned, by, C_):
    """C == Cs in {32, 64} would take the fused kernel (float4 loads of x, w1, w2, b1, b2, float4 stores of out); with any
    of them off a 16-byte boundary the call goes to the two-launch path, which reports the missing tmp"""
    rc = _call_cl(_ptrs(misaligned, by), C_, C_)
    assert rc != 0
    msg = _error()
    assert "tmp" in msg and "16-byte aligned" in msg, msg


@pytest.mark.parametrize("C_", [32, 64])
@pytest.mark.parametrize("T", [1, 127, 128, 5000])
@pytest.mark.parametrize("misaligned,by", [("x", 4), ("x", 8), ("out", 4), ("out", 8), ("b1", 4), ("b2", 4)])
def test_resblock_tc_rejects_misaligned_pointers(misaligned, by, T, C_):
    """x / out 16-byte and b1 / b2 8-byte alignment, on both sides of the T = 128 split between the two kernels"""
    rc = _call_tc(_ptrs(misaligned, by), C_, T)
    assert rc != 0
    msg = _error()
    assert msg.startswith("jk_resblock_tc:") and "x and out must be 16-byte aligned" in msg and "8-byte aligned" in msg, msg


def test_resblock_tc_checks_alignment_before_the_channel_count():
    """an unsupported C with misaligned pointers reports the pointers (the first constraint checked), still without a
    launch; with aligned pointers the channel count is what fails"""
    rc = _call_tc(_ptrs("x", 4), 48, 300)
    assert rc != 0 and "16-byte aligned" in _error()
    rc = _call_tc(_ptrs(None, 0), 48, 300)
    assert rc != 0 and "C must be 32 or 64" in _error()


def test_resblock_signatures_take_integer_addresses():
    """the ctypes mirrors accept plain integers for device pointers, as the GPU tests pass them"""
    from jukebox_b200 import _lib
    res, args = _lib.SIGNATURES["jk_resblock_cl"]
    assert res is C.c_int and args[:7] == [C.c_void_p] * 7
    res, args = _lib.SIGNATURES["jk_resblock_tc"]
    assert res is C.c_int and args[:6] == [C.c_void_p] * 6
