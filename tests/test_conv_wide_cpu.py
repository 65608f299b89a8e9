"""CPU checks of the wide tensor-core convolutions (jk_conv1d_tc_wide): the library exports the new entry points with the
ctypes signatures of jukebox_b200/_lib.py, the split-precision TMA kernels (vqvae_t5.cu, score.cu) use no stack and do
not spill (nvcc -Xptxas -v for sm_90a), and only the
decoder side of a VQ-VAE sets `tensor_cores` (the encoder's output feeds the bit-exact codebook argmin)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = {
    "jk_conv_weight_split_bytes": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]),
    "jk_pack_conv_weight_split": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                 ctypes.c_void_p]),
}


def test_new_symbols_are_exported_with_their_signatures():
    from jukebox_b200 import _lib
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name, (res, args) in NEW.items():
        assert hasattr(handle, name), name
        assert _lib.SIGNATURES[name] == (res, args), name
    res, args = _lib.SIGNATURES["jk_conv1d_tc_wide"]
    assert hasattr(handle, "jk_conv1d_tc_wide")
    assert res is ctypes.c_int and args[1:] == [ctypes.c_void_p, ctypes.c_void_p]
    assert args[0]._type_ is _lib.ConvArgs


def test_split_byte_count():
    from jukebox_b200 import _lib
    n = ctypes.c_size_t(0)
    assert _lib.lib().jk_conv_weight_split_bytes(3, 1920, 1024, ctypes.byref(n)) == 0
    assert n.value == 2 * 3 * 1920 * 1024 * 2                       # hi and lo planes of fp16
    assert _lib.lib().jk_conv_weight_split_bytes(0, 64, 64, ctypes.byref(n)) != 0


# the split-precision TMA kernels of each source and how many instantiations of each it compiles
SPLIT_TMA_KERNELS = {
    "vqvae_t5.cu": {"conv_wide_kernel": 2, "conv_t5_kernel": 4, "resblock_t5_kernel": 2, "pack_split_kernel": 1},
    "score.cu": {"xout_head_kernel": 2},
}


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"),
                    reason="needs the CUDA toolkit")
def test_wide_conv_kernels_do_not_spill(tmp_path):
    from jukebox_b200.build import _nvcc
    for source, kernels in SPLIT_TMA_KERNELS.items():
        src = os.path.join(ROOT, "jukebox_b200", "csrc", source)
        cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
               "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "kernels.o"), "-I", os.path.join(ROOT, "include")]
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-3000:]
        report = {}
        current = None
        for line in out.stderr.splitlines():
            m = re.search(r"Compiling entry function '(\w+)'", line)
            if m:
                current = m.group(1)
                continue
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m and current:
                report[current] = tuple(int(v) for v in m.groups())
        for kernel, count in kernels.items():
            found = {k: v for k, v in report.items() if kernel in k}
            assert len(found) == count, (source, kernel, report)
            for name, (stack, st, ld) in found.items():
                assert stack == 0 and st == 0 and ld == 0, f"{name}: {stack} bytes stack, spills {st} bytes / loads {ld} bytes"


def test_only_the_decoder_side_sets_tensor_cores():
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae
    vq = make_vqvae(setup_hparams("small_vqvae", dict(restore_vqvae="", sample_length=8192)), "cpu")
    enc = [m for m in vq.encoders.modules() if hasattr(m, "tensor_cores")]
    dec = [m for m in vq.decoders.modules() if hasattr(m, "tensor_cores")]
    assert enc and dec
    assert not any(m.tensor_cores for m in enc)
    blocks = [m for d in vq.decoders for m in d.level_blocks.modules() if hasattr(m, "tensor_cores")]
    assert blocks and all(m.tensor_cores for m in blocks)
