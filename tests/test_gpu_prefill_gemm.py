"""wgmma + TMA prefill Conv1D (jk_conv1d_prefill_f16) against an fp32 torch reference of the same op."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def run(M, N, K, seed, bias=True):
    from jukebox_b200._lib import lib, check, ptr, stream_ptr
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, generator=g, device="cuda").half()
    w = (torch.randn(K, N, generator=g, device="cuda") / K ** 0.5).half()       # Conv1D.w layout [n_in, n_out]
    b = torch.randn(N, generator=g, device="cuda") if bias else None
    w_t = w.t().contiguous()
    y = torch.empty(M, N, dtype=torch.float16, device="cuda")
    check(lib().jk_conv1d_prefill_f16(ptr(x), ptr(w_t), ptr(b), ptr(y), M, N, K, stream_ptr()))
    ref = x.float() @ w.float() + (b if bias else 0)
    torch.cuda.synchronize()
    err = (y.float() - ref).abs().max().item() / ref.abs().max().item()
    return err


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 128, 256), (256, 384, 512), (300, 200, 192),
                                   (1, 8, 64), (4096, 2400, 4800),
                                   # K tails (TMA zero-fills beyond K): released-upsampler n_state 480, 5b n_state 1200
                                   (256, 1920, 480), (200, 4800, 1200), (130, 136, 72)])
def test_prefill_gemm_matches_fp32_reference(M, N, K):
    err = run(M, N, K, seed=M + N + K)
    print(f"prefill GEMM M={M} N={N} K={K}: rel err {err:.2e}")
    assert err < 2e-3        # fp16 output rounding (2^-11 of the value) + fp32 accumulation order


def test_prefill_gemm_no_bias_and_determinism():
    a = run(384, 256, 128, seed=7, bias=False)
    b = run(384, 256, 128, seed=7, bias=False)
    assert a == b and a < 2e-3
