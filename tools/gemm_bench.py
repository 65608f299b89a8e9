"""Throughput of the wgmma prefill Conv1D at the 5b_lyrics c_enc_kv shape (and a square shape), CUDA events."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from jukebox_b200._lib import lib, check, ptr, stream_ptr  # noqa: E402

peaks = {}
try:
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
except Exception:
    pass
peak = float(peaks.get("bf16_tflops", 1590.0))
for (M, N, K) in [(4096, 2400, 4800), (8192, 8192, 8192), (16384, 4800, 4800)]:
    x = torch.randn(M, K, device="cuda").half()
    wt = torch.randn(N, K, device="cuda").half()
    b = torch.randn(N, device="cuda")
    y = torch.empty(M, N, dtype=torch.float16, device="cuda")
    for _ in range(3):
        check(lib().jk_conv1d_prefill_f16(ptr(x), ptr(wt), ptr(b), ptr(y), M, N, K, stream_ptr()))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps):
        check(lib().jk_conv1d_prefill_f16(ptr(x), ptr(wt), ptr(b), ptr(y), M, N, K, stream_ptr()))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
    print(f"jk_conv1d_prefill_f16 M={M} N={N} K={K}: {ms * 1e3:.1f} us, {tf:.1f} TFLOP/s = {tf / peak:.3f} of measured cuBLAS bf16 peak ({peak:.0f})")
