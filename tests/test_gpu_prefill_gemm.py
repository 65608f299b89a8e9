"""wgmma + TMA prefill Conv1D (jk_conv1d_prefill_f16, jk_prefill_gemm_f16) against torch references of the same op.

The exact-grid tests make x and w small integers over powers of two, so that the fp32 accumulation is exact in any order:
the reference is then the float64 product followed by the epilogue's own float32 / fp16 steps in the order
epilogue_value (prefill_gemm.cu) applies them:
  y = fp16(acc + bias)                       (fp32 add)
  epi 0: y;  epi 2: fp16(res + y);  epi 1: z = fp16(1.702 y), sg = fp16(1 / (1 + exp(-z))), out = fp16(y sg)
Epilogues 0 and 2 must match bitwise; epilogue 1 within one fp16 ulp per element (the device expf is not torch's exp).
Shapes cover M and N at the 128-wide tile edges, odd N (scalar stores and scalar residual reads), one K block, K tails,
exactly STAGES (3) blocks and the ring wrapping many times; a guard after y must be unchanged."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 512


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


# ---- exact grid: every epilogue, bitwise --------------------------------------------------------------------------------
def grid(shape, lim, scale, g):
    """integers in [-lim, lim] times 2^-scale, fp16-exact"""
    return (torch.randint(-lim, lim + 1, shape, generator=g, device="cuda").double() * 2.0 ** -scale).half()


def epilogue_ref(acc, bias, res, epi):
    """epilogue_value on float64-exact accumulators, with the kernel's float32 operations"""
    y = acc.float()
    if bias is not None:
        y = y + bias[None, :]
    y = y.half().float()
    if epi == 0:
        return y.half()
    if epi == 2:
        return (res.float() + y).half()
    z = (y * torch.tensor(1.702, dtype=torch.float32, device="cuda")).half().float()
    sg = (1.0 / (1.0 + torch.exp(-z))).half().float()
    return (y * sg).half()


def gemm(x, w_t, bias, res, M, N, K, epi, g):
    """jk_prefill_gemm_f16 into a NaN-filled y followed by a guard pattern -> y [M, N]; asserts the guard is intact"""
    from jukebox_b200._lib import lib, ptr, stream_ptr
    buf = torch.full((M * N + GUARD,), float("nan"), dtype=torch.float16, device="cuda")
    buf[M * N:] = torch.randn(GUARD, generator=g, device="cuda").half()
    guard = buf[M * N:].clone()
    rc = lib().jk_prefill_gemm_f16(ptr(x), ptr(w_t), ptr(bias), ptr(res), buf.data_ptr(), M, N, K, epi, stream_ptr())
    assert rc == 0, lib().jk_last_error().decode()
    torch.cuda.synchronize()
    assert torch.equal(buf[M * N:], guard), f"M {M} N {N} K {K} epi {epi}: store past the end of y"
    return buf[:M * N].view(M, N)


def fp16_ulp(x):
    a = x.double().abs()
    _, e = torch.frexp(a)
    return torch.where(a < 2.0 ** -14, torch.full_like(a, 2.0 ** -24), torch.ldexp(torch.ones_like(a), e - 11))


KS = (64, 72, 192, 200, 480, 1200, 4800)


@pytest.mark.parametrize("N", [8, 127, 128, 129, 2401])
@pytest.mark.parametrize("M", [1, 127, 128, 129, 300])
def test_prefill_gemm_epilogues_exact_grid(M, N):
    """x: integers in [-8, 8] / 8, w: integers in [-8, 8] / 64; |partial sums| <= 4800 / 8 in units of 2^-9, far below
    2^24 of them, so the accumulation is exact in fp32.  Bias on even M, NULL on odd M."""
    g = torch.Generator(device="cuda").manual_seed(1000 * M + N)
    not_bitwise = []
    for K in KS:
        x = grid((M, K), 8, 3, g)
        w_t = grid((N, K), 8, 6, g)
        bias = (torch.randn(N, generator=g, device="cuda") * 4).half().float() if M % 2 == 0 else None
        res = torch.randn(M, N, generator=g, device="cuda").half()
        acc = x.double() @ w_t.double().t()
        for epi in (0, 1, 2):
            y = gemm(x, w_t, bias, res if epi == 2 else None, M, N, K, epi, g)
            ref = epilogue_ref(acc, bias, res, epi)
            assert not torch.isnan(y).any(), f"M {M} N {N} K {K} epi {epi}: element not written"
            if epi == 1:
                d = (y.double() - ref.double()).abs()
                bad = d > fp16_ulp(ref)
                assert not bad.any(), (f"M {M} N {N} K {K} quick_gelu: {int(bad.sum())} elements beyond one fp16 ulp, "
                                       f"first at {bad.nonzero()[0].tolist()}")
                not_bitwise.append(float((y != ref).double().mean()))
            else:
                diff = y != ref
                assert not diff.any(), (f"M {M} N {N} K {K} epi {epi}: {int(diff.sum())} elements differ, first at "
                                        f"{diff.nonzero()[0].tolist()}: {y[diff][0].item()} vs {ref[diff][0].item()}")
    print(f"M {M} N {N}: quick_gelu elements not bitwise equal: at most {max(not_bitwise):.2e} of a call")
