"""Every kernel route of the VQ-VAE's small-channel convolutions against float64, at its tile and pipeline edges.

jk_conv1d_cl, jk_resblock_cl and jk_resblock_tc choose between eight kernels by shape, flag and pointer alignment
(vqvae_kernels.cu, vqvae_t5.cu).  Each case here names the route it targets, and `expected_route` mirrors that dispatch,
so a change to it fails a route assertion instead of silently moving the coverage elsewhere.  The reference is the
formula of jk_conv_args in jkb200.h, written as a float64 gather:

    out[t * os + oo] = res + scale * (bias + sum_tap W[tap]^T . pre(in[t * in_stride + off_tap]))

Bounds against it: 2e-6 of max |ref| for the exact fp32-FMA kernels, 4e-6 for the split-precision tensor-core ones.
The exact kernels share one FMA order (tap, then input channel), which the encoder relies on: its output feeds the
bit-exact codebook argmin, and which exact kernel runs depends on alignment and a shared-memory cutoff.  So the narrow,
tile and fused kernels are also compared with the generic kernel (forced by an input 4 bytes off a 16-byte boundary, which
it reads with scalar loads): bitwise without a residual, and within one fp32 rounding of the residual sum with one."""
import ctypes as C
import math
import zlib
from dataclasses import dataclass, field

import pytest
import torch

from jukebox_b200 import _lib
from jukebox_b200._lib import lib, stream_ptr

pytestmark = pytest.mark.gpu

EXACT_TOL, TC_TOL = 2e-6, 4e-6
K4S2 = [-1, 0, 1, 2]                       # Conv1d(k4, s2, p1) taps on the stride-2 input
PHASES = (([0, -1], 0), ([1, 0], 1))       # the two phases of ConvTranspose1d(k4, s2, p1): (taps, output row offset)


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ---- the dispatch, mirrored --------------------------------------------------------------------------------------------
def expected_route(a):
    """the kernel jk_conv1d_cl picks for ConvArgs `a` (vqvae_kernels.cu)"""
    p = lambda v: v or 0
    if (a.c_out <= 4 and a.c_in % 4 == 0 and a.c_in <= 128 and p(a.inp) % 16 == 0
            and a.n_taps * a.c_in * a.c_out * 4 <= 32768):
        return "narrow"
    vec = (p(a.inp) | p(a.out) | p(a.bias) | p(a.res)) % 16 == 0
    if a.tensor_cores and a.c_in in (32, 64) and a.c_out in (32, 64) and vec:
        return "t5" if a.in_stride == 1 and a.n_taps <= 3 and a.t_in >= 128 and a.t_out >= 1 else "h2"
    if a.c_out in (32, 64) and a.c_in % 4 == 0 and 4 <= a.c_in <= 64 and vec and p(a.w) % 16 == 0:
        tt = 8 * 256 // (a.c_out // 4)                    # positions per CTA: 128 for c_out 64, 256 for c_out 32
        if (a.n_taps * a.c_in * a.c_out + a.n_taps * tt * (a.c_in + 4)) * 4 <= 220 * 1024:
            return f"tile{a.c_out}"
    return "generic"


def expected_resblock_cl_route(x, out, w1, b1, w2, b2, C_, Cs, T):
    ptrs = [t.data_ptr() for t in (x, out, w1, b1, w2, b2)]
    if C_ == Cs and C_ in (32, 64) and x.data_ptr() != out.data_ptr() and T > 0 and all(v % 16 == 0 for v in ptrs):
        return "fused"
    return "two-launch"


def expected_resblock_tc_route(T):
    return "t5" if T >= 128 else "h2"


# ---- calls ---------------------------------------------------------------------------------------------------------------
def _p(t):
    return None if t is None else t.data_ptr()


def conv(x, w, bias, t_out, taps, *, out, in_stride=1, out_stride=1, out_offset=0, relu_in=False, scale=1.0, res=None,
         tc=False, route=None):
    """jk_conv1d_cl on [n, t_in, c_in] -> rows t * out_stride + out_offset of out, filled as ops_cl._conv does"""
    n, t_in, c_in = x.shape
    a = _lib.ConvArgs()
    a.inp, a.t_in, a.c_in = _p(x), t_in, c_in
    a.out, a.t_out, a.c_out = _p(out), t_out, w.shape[2]
    a.w, a.bias, a.res = _p(w), _p(bias), _p(res)
    a.n_taps = len(taps)
    for i, o in enumerate(taps):
        a.tap_off[i] = int(o)
    a.in_stride, a.out_stride, a.out_offset = in_stride, out_stride, out_offset
    a.relu_in, a.scale, a.n, a.tensor_cores = int(relu_in), float(scale), n, int(tc)
    got = expected_route(a)
    assert route is None or got == route, f"dispatch takes {got}, the case targets {route}"
    rc = lib().jk_conv1d_cl(C.byref(a), stream_ptr())
    assert rc == 0, lib().jk_last_error().decode()
    return got


def resblock_cl(x, out, tmp, w1, b1, w2, b2, T, C_, Cs, dil, rs):
    rc = lib().jk_resblock_cl(_p(x), _p(out), _p(tmp), _p(w1), _p(b1), _p(w2), _p(b2), x.shape[0], T, C_, Cs, dil, rs,
                              stream_ptr())
    assert rc == 0, lib().jk_last_error().decode()


def resblock_tc(x, out, w1, b1, w2, b2, T, C_, dil, rs):
    rc = lib().jk_resblock_tc(_p(x), _p(out), _p(w1), _p(b1), _p(w2), _p(b2), x.shape[0], T, C_, dil, rs, stream_ptr())
    assert rc == 0, lib().jk_last_error().decode()


def misaligned(x):
    """x's values in a flat buffer viewed from element 1: 4-byte aligned, not 16"""
    buf = torch.empty(x.numel() + 1, device=x.device, dtype=x.dtype)
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 16 == 4
    return v


# ---- float64 references --------------------------------------------------------------------------------------------------
def conv_ref(x, w, bias, t_out, taps, in_stride=1, relu_in=False, scale=1.0, res=None):
    """the jk_conv_args formula as a gather: [n, t_out, c_out] float64, rows outside [0, t_in) read as zero"""
    x = x.double()
    if relu_in:
        x = x.clamp_min(0)
    n, t_in, _ = x.shape
    t = torch.arange(t_out, device=x.device)
    acc = torch.zeros(n, t_out, w.shape[2], dtype=torch.float64, device=x.device)
    for j, off in enumerate(taps):
        pos = t * in_stride + off
        ok = ((pos >= 0) & (pos < t_in)).double()[None, :, None]
        acc += (x[:, pos.clamp(0, t_in - 1)] * ok) @ w[j].double()
    if bias is not None:
        acc += bias.double()
    y = scale * acc
    return y if res is None else y + res.double()


def block_ref(x, w1, b1, w2, b2, dil, rs):
    """ResConv1DBlock: x + rs * (W2 . relu(W1 *_dil relu(x) + b1) + b2)"""
    T = x.shape[1]
    h = conv_ref(x, w1, b1, T, [-dil, 0, dil], relu_in=True)
    return conv_ref(h, w2, b2, T, [0], relu_in=True, scale=rs, res=x)


def rel_err(out, ref):
    return float((out.double() - ref).abs().max() / ref.abs().max())


def _ulp(v):
    """spacing of fp32 numbers at |v| (float64), subnormal floor included"""
    _, e = torch.frexp(v.float().abs())
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), (e - 24).clamp(min=-149))


def same_up_to_residual_rounding(a, b, res_rows):
    """a and b agree bitwise, or differ only by the one rounding of scale * y that an FMA-contracted residual add skips
    (fl(fl(s y) + r) against fl(s y + r)): within ulp(s y) + ulp(result) elementwise.  Returns whether bitwise."""
    if torch.equal(a, b):
        return True
    pre = (a.double() - res_rows.double()).abs()
    tol = _ulp(pre) + _ulp(torch.maximum(a.abs(), b.abs()))
    diff = (a.double() - b.double()).abs()
    assert bool((diff <= tol).all()), f"max difference {float(diff.max()):.3e} beyond one rounding of the residual sum"
    return False


# ---- cases ---------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    route: str
    ci: int
    co: int
    T: int                                  # output positions per call (per phase)
    taps: list = field(default_factory=lambda: [-1, 0, 1])
    n: int = 1
    stride: int = 1
    relu: bool = False
    scale: float = 1.0
    res: bool = False
    bias: bool = True
    phases: bool = False                    # both ConvTranspose1d phases into one [n, 2T, co] buffer
    ostride: tuple = (1, 0)                 # (out_stride, out_offset) of a single call

    def __str__(self):
        taps = "phases" if self.phases else "taps" + ",".join(map(str, self.taps)) + (f" s{self.stride}" if self.stride > 1 else "")
        extra = "".join([" relu" if self.relu else "", f" res*{self.scale}" if self.res else
                         (f" *{self.scale}" if self.scale != 1 else ""), "" if self.bias else " nobias",
                         f" os{self.ostride[0]}+{self.ostride[1]}" if self.ostride != (1, 0) else ""])
        return f"{self.route} {self.ci}->{self.co} T{self.T} n{self.n} {taps}{extra}"


def _setup(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    x = rnd(c.n, c.T * c.stride, c.ci)
    if c.phases:
        calls = [(rnd(2, c.ci, c.co) / math.sqrt(2 * c.ci), taps, oo) for taps, oo in PHASES]
        os_ = 2
    else:
        k = len(c.taps)
        calls = [(rnd(k, c.ci, c.co) / math.sqrt(k * c.ci), c.taps, c.ostride[1])]
        os_ = c.ostride[0]
    bias = rnd(c.co) * 0.1 if c.bias else None
    res = rnd(c.n, c.T * os_, c.co) if c.res else None
    return x, calls, bias, res, os_


def _run(c, x, calls, bias, res, os_, tc, route):
    out = torch.full((c.n, c.T * os_, c.co), float("nan"), device="cuda")
    for w, taps, oo in calls:
        conv(x, w, bias, c.T, taps, out=out, in_stride=c.stride, out_stride=os_, out_offset=oo, relu_in=c.relu,
             scale=c.scale, res=res, tc=tc, route=route)
    return out


def _ref(c, x, calls, bias, res, os_):
    """[n, T * os, co] float64; rows no call writes are nan"""
    ref = torch.full((c.n, c.T * os_, c.co), float("nan"), dtype=torch.float64, device="cuda")
    for w, taps, oo in calls:
        ref[:, oo::os_] = conv_ref(x, w, bias, c.T, taps, in_stride=c.stride, relu_in=c.relu, scale=c.scale,
                                   res=None if res is None else res[:, oo::os_])
    return ref


def _check(c, out, ref, tol):
    torch.cuda.synchronize()
    written = ~torch.isnan(ref)
    assert torch.equal(torch.isnan(out), ~written), "rows outside the call's phase were written, or rows were missed"
    e = rel_err(out[written], ref[written])
    return e, e < tol


NARROW = [
    Case("narrow", 64, 1, 5000, n=3),                                            # Decoder.out: 64 -> 1 audio channel
    Case("narrow", 64, 1, 257, relu=True, res=True, scale=0.25),
    Case("narrow", 4, 2, 255, [-8, 0, 8], n=3),                                  # span 16: the staged-window limit
    Case("narrow", 12, 3, 256, [-9, 0, 9], relu=True),                           # span 18: tap by tap
    Case("narrow", 100, 4, 257, [-27, 0, 27], n=3, res=True, scale=0.7, ostride=(2, 1)),
    Case("narrow", 128, 4, 255, K4S2, stride=2),                                 # stride 2: tap by tap
    Case("narrow", 128, 1, 1, K4S2, n=3, stride=2, relu=True, res=True, scale=0.25),
    Case("narrow", 64, 2, 1, [0], ostride=(2, 0)),
    Case("narrow", 12, 1, 5000, [-8, 0, 8], relu=True, res=True, scale=0.7),
    Case("narrow", 100, 3, 256, n=3),
    Case("narrow", 4, 4, 1, [-27, 0, 27], relu=True, res=True, scale=0.25, bias=False),
    Case("narrow", 128, 2, 5000, [-9, 0, 9], n=3, relu=True, ostride=(2, 0)),
    Case("narrow", 64, 4, 257, K4S2, stride=2, res=True, scale=0.7),
    Case("narrow", 100, 1, 255, [-1, 0, 1, 2], n=1, relu=True),                  # 4 taps, stride 1, one window
]

TILE = [
    Case("tile64", 4, 64, 127, n=2),                                             # tile height 128 for c_out 64
    Case("tile64", 36, 64, 128, [-27, 0, 27], relu=True, res=True, scale=0.7),
    Case("tile64", 64, 64, 129, K4S2, n=3, stride=2),
    Case("tile64", 64, 64, 128, n=2, phases=True),
    Case("tile64", 4, 64, 129, phases=True, res=True, scale=0.25),
    Case("tile64", 36, 64, 127, K4S2, stride=2, relu=True, bias=False),
    Case("tile32", 4, 32, 255, [-27, 0, 27], res=True, scale=0.25),              # tile height 256 for c_out 32
    Case("tile32", 36, 32, 256, K4S2, n=2, stride=2, relu=True),
    Case("tile32", 64, 32, 257, n=3, phases=True, res=True, scale=0.7),
    Case("tile32", 36, 32, 257, [-1, 0, 1]),
    Case("tile32", 64, 32, 256, [-3, 0]),
    Case("tile32", 4, 32, 255, K4S2, stride=2, relu=True, res=True, scale=0.7),
]

GENERIC = [
    Case("generic", 64, 32, 300, K4S2, n=2, stride=2),                           # 311 KB of shared memory: over the cutoff
    Case("generic", 64, 32, 257, [-1, 0, 1], relu=True, res=True, scale=0.7),     # 233 KB: over the cutoff
    Case("generic", 1, 64, 64, K4S2, n=2, stride=2),                             # the encoder input conv
    Case("generic", 3, 5, 63, n=3, relu=True, res=True, scale=0.7),
    Case("generic", 33, 48, 65, [-3, 0, 3]),                                     # ragged input-channel slab
    Case("generic", 96, 96, 64, K4S2, n=2, stride=2, relu=True, res=True, scale=0.25),
    Case("generic", 130, 130, 65, n=1, res=True, scale=0.7),                     # 5 slabs, 3 column tiles
    Case("generic", 96, 130, 63, [-2187, 0, 2187], bias=False),
    Case("generic", 130, 5, 64, phases=True, relu=True),
    Case("generic", 1, 48, 65, [0], ostride=(2, 1)),
]


@pytest.mark.parametrize("c", NARROW + TILE + GENERIC, ids=str)
def test_exact_conv_matches_fp64(c):
    args = _setup(c, zlib.crc32(str(c).encode()) % 1000)
    out = _run(c, *args, tc=False, route=c.route)
    e, ok = _check(c, out, _ref(c, *args), EXACT_TOL)
    print(f"{c}: {e:.1e} vs fp64")
    assert ok, e


@pytest.mark.parametrize("c", NARROW + TILE, ids=str)
def test_exact_routes_agree_with_the_generic_kernel(c):
    """the narrow and tile kernels against the generic kernel on the same values: bitwise without a residual, one
    rounding of the residual sum with one"""
    x, calls, bias, res, os_ = _setup(c, zlib.crc32(str(c).encode()) % 1000)
    out = _run(c, x, calls, bias, res, os_, tc=False, route=c.route)
    gen = _run(c, misaligned(x), calls, bias, res, os_, tc=False, route="generic")
    torch.cuda.synchronize()
    written = ~torch.isnan(out)
    assert torch.equal(written, ~torch.isnan(gen))
    if res is None:
        assert torch.equal(out[written], gen[written])
        print(f"{c}: bitwise equal to the generic kernel")
    else:
        bitwise = same_up_to_residual_rounding(out[written], gen[written], res[written])
        print(f"{c}: {'bitwise equal to' if bitwise else 'within one rounding of the residual sum of'} the generic kernel")


# ---- exact residual block ------------------------------------------------------------------------------------------------
def _block_weights(C_, Cs, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    return (rnd(3, C_, Cs) / math.sqrt(3 * C_), rnd(Cs) * 0.1, rnd(1, Cs, C_) / math.sqrt(Cs), rnd(C_) * 0.1)


@pytest.mark.parametrize("C_", [32, 64])
@pytest.mark.parametrize("T", [1, 127, 128, 129, 255, 256, 257, 4101])
def test_fused_resblock_matches_its_two_launch_form_and_fp64(T, C_):
    """jk_resblock_cl's fused kernel against the two jk_conv1d_cl launches it stands for (k3 with relu_in into tmp, then
    k1 with relu_in, res = x and scale = res_scale into a separate out) and against fp64"""
    n = 2
    for dil in (1, 3, 2187):
        for rs in (1.0, 0.25, 0.7):
            w1, b1, w2, b2 = _block_weights(C_, C_, T + dil)
            x = torch.randn(n, T, C_, device="cuda")
            fused = torch.empty_like(x)
            assert expected_resblock_cl_route(x, fused, w1, b1, w2, b2, C_, C_, T) == "fused"
            resblock_cl(x, fused, None, w1, b1, w2, b2, T, C_, C_, dil, rs)
            tmp, two = torch.empty_like(x), torch.empty_like(x)
            conv(x, w1, b1, T, [-dil, 0, dil], out=tmp, relu_in=True, route=f"tile{C_}")
            conv(tmp, w2, b2, T, [0], out=two, relu_in=True, res=x, scale=rs, route=f"tile{C_}")
            ref = block_ref(x, w1, b1, w2, b2, dil, rs)
            torch.cuda.synchronize()
            e_f, e_t = rel_err(fused, ref), rel_err(two, ref)
            bitwise = same_up_to_residual_rounding(fused, two, x)
            print(f"C {C_} T {T} dil {dil} rs {rs}: fused {e_f:.1e}, two-launch {e_t:.1e} vs fp64; "
                  f"{'bitwise equal' if bitwise else 'within one rounding of the residual sum'}")
            assert e_f < EXACT_TOL and e_t < EXACT_TOL, (e_f, e_t)


@pytest.mark.parametrize("C_,Cs", [(64, 32), (32, 128)])
@pytest.mark.parametrize("T", [129, 1000])
def test_resblock_cl_through_tmp_matches_fp64(C_, Cs, T):
    w1, b1, w2, b2 = _block_weights(C_, Cs, C_ + Cs + T)
    x = torch.randn(2, T, C_, device="cuda")
    out, tmp = torch.empty_like(x), torch.empty(2, T, Cs, device="cuda")
    assert expected_resblock_cl_route(x, out, w1, b1, w2, b2, C_, Cs, T) == "two-launch"
    resblock_cl(x, out, tmp, w1, b1, w2, b2, T, C_, Cs, 3, 0.7)
    e = rel_err(out, block_ref(x, w1, b1, w2, b2, 3, 0.7))
    print(f"C {C_} Cs {Cs} T {T}: {e:.1e} vs fp64")
    assert e < EXACT_TOL


@pytest.mark.parametrize("C_", [32, 64])
def test_resblock_with_misaligned_x(C_):
    """x 4 bytes off a 16-byte boundary: jk_resblock_cl runs its two-launch path through tmp (the generic kernel) and
    equals the fused call on an aligned copy; without tmp, and on jk_resblock_tc, it is an error and nothing runs"""
    T, dil, rs = 257, 3, 0.7
    w1, b1, w2, b2 = _block_weights(C_, C_, C_)
    x = torch.randn(2, T, C_, device="cuda")
    xm = misaligned(x)
    ref_out, out, tmp = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    assert expected_resblock_cl_route(xm, out, w1, b1, w2, b2, C_, C_, T) == "two-launch"
    resblock_cl(x, ref_out, None, w1, b1, w2, b2, T, C_, C_, dil, rs)
    resblock_cl(xm, out, tmp, w1, b1, w2, b2, T, C_, C_, dil, rs)
    torch.cuda.synchronize()
    bitwise = same_up_to_residual_rounding(out, ref_out, x)
    print(f"C {C_}: misaligned x {'bitwise equal to' if bitwise else 'within one rounding of'} the aligned fused call")
    assert rel_err(out, block_ref(x, w1, b1, w2, b2, dil, rs)) < EXACT_TOL
    assert lib().jk_resblock_cl(_p(xm), _p(out), None, _p(w1), _p(b1), _p(w2), _p(b2), 2, T, C_, C_, dil, rs,
                                stream_ptr()) != 0
    assert lib().jk_resblock_tc(_p(xm), _p(out), _p(w1), _p(b1), _p(w2), _p(b2), 2, T, C_, dil, rs, stream_ptr()) != 0
    assert "16-byte aligned" in lib().jk_last_error().decode()


# ---- tensor-core convolutions --------------------------------------------------------------------------------------------
PAIRS = [(32, 32), (32, 64), (64, 32), (64, 64)]
T5_CASES = [c for ci, co in PAIRS for c in (
    Case("t5", ci, co, 128),
    Case("t5", ci, co, 129, [0], relu=True, res=True, scale=0.7),                # 1 tap
    Case("t5", ci, co, 255, [-2187, 0, 2187], n=2, bias=False),
    Case("t5", ci, co, 256, n=2, phases=True),                                   # out_stride-2 phases, 2 taps
    Case("t5", ci, co, 257, [-3, 5], relu=True, res=True, scale=0.25),
    Case("t5", ci, co, 1000, [-27, 0, 27], n=3, relu=True, res=True, scale=0.7, bias=False),
)]
H2_CASES = [c for ci, co in PAIRS for c in (
    Case("h2", ci, co, 1, n=3),
    Case("h2", ci, co, 15, relu=True, res=True, scale=0.7),
    Case("h2", ci, co, 16, [0], bias=False),
    Case("h2", ci, co, 17, n=2, phases=True, res=True, scale=0.25),
    Case("h2", ci, co, 127, [-27, 0, 27], n=2, relu=True),
    Case("h2", ci, co, 127, K4S2, n=2, stride=2, res=True, scale=0.7),           # stride 2, 4 taps
    Case("h2", ci, co, 100, K4S2, n=1, stride=2, relu=True, bias=False),
)]


@pytest.mark.parametrize("c", T5_CASES + H2_CASES, ids=str)
def test_tensor_core_conv_matches_fp64(c):
    args = _setup(c, zlib.crc32(str(c).encode()) % 1000)
    out = _run(c, *args, tc=True, route=c.route)
    e, ok = _check(c, out, _ref(c, *args), TC_TOL)
    print(f"{c}: {e:.1e} vs fp64")
    assert ok, e


@pytest.mark.parametrize("ci,co", PAIRS)
@pytest.mark.parametrize("kind", ["k3", "phases"])
def test_t5_conv_under_load(kind, ci, co):
    """at least four tiles per CTA, so that every ring stage and barrier phase of conv_t5_kernel turns over several times"""
    n, sms = 4, _sms()
    T = 128 * -(-4 * _sms() // n) + 37
    assert n * -(-T // 128) >= 4 * sms
    c = Case("t5", ci, co, T, [-1, 0, 1], n=n, relu=kind == "k3", phases=kind == "phases", res=True, scale=0.7)
    args = _setup(c, ci + co)
    out = _run(c, *args, tc=True, route="t5")
    e, ok = _check(c, out, _ref(c, *args), TC_TOL)
    print(f"{c}: {e:.1e} vs fp64, {n * -(-T // 128)} tiles on {sms} SMs")
    assert ok, e


@pytest.mark.parametrize("ci,co", PAIRS)
def test_h2_conv_with_more_than_16_tiles_per_sm(ci, co):
    """stride 2, n = 8, 5000 outputs: more 16-position tiles than the 16 warps of every CTA, so each warp runs the
    cross-tile prefetch of its next tile"""
    sms = _sms()
    c = Case("h2", ci, co, 5000, K4S2, n=8, stride=2, relu=True, res=True, scale=0.7)
    assert c.n * -(-c.T // 16) > 16 * sms
    args = _setup(c, ci * co)
    out = _run(c, *args, tc=True, route="h2")
    e, ok = _check(c, out, _ref(c, *args), TC_TOL)
    print(f"{c}: {e:.1e} vs fp64")
    assert ok, e


# ---- tensor-core residual block ------------------------------------------------------------------------------------------
def _tc_block_case(C_, T, n, dil, rs=0.7):
    w1, b1, w2, b2 = _block_weights(C_, C_, C_ + T + dil)
    x = torch.randn(n, T, C_, device="cuda")
    out = torch.empty_like(x)
    resblock_tc(x, out, w1, b1, w2, b2, T, C_, dil, rs)
    return rel_err(out, block_ref(x, w1, b1, w2, b2, dil, rs))


@pytest.mark.parametrize("C_", [32, 64])
@pytest.mark.parametrize("T", [128, 129, 255, 256, 257])
def test_t5_resblock_matches_fp64(T, C_):
    """more tiles than SMs; dilations inside the tile, across it and beyond the clip"""
    assert expected_resblock_tc_route(T) == "t5"
    n = 2 * _sms() // -(-T // 128) + 1
    for dil in (1, 27, T + 5):
        e = _tc_block_case(C_, T, n, dil)
        print(f"t5 block C {C_} T {T} n {n} dil {dil}: {e:.1e} vs fp64")
        assert e < TC_TOL, e


@pytest.mark.parametrize("C_", [32, 64])
@pytest.mark.parametrize("T", [1, 17, 127])
def test_h2_resblock_matches_fp64(T, C_):
    """more 16-position tiles than 16 x SMs, so every warp runs a second tile"""
    assert expected_resblock_tc_route(T) == "h2"
    n = 16 * _sms() // -(-T // 16) + 1
    for dil in (1, 9, T + 3):
        e = _tc_block_case(C_, T, n, dil)
        print(f"h2 block C {C_} T {T} n {n} dil {dil}: {e:.1e} vs fp64")
        assert e < TC_TOL, e


# ---- invariants ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route,T", [("t5", 5000), ("h2", 127)])
@pytest.mark.parametrize("ci,co", [(32, 64), (64, 64)])
def test_tensor_core_conv_clip_alone_equals_clip_in_batch(route, T, ci, co):
    n = 6 if route == "t5" else 300
    c = Case(route, ci, co, T, [-3, 0, 3], n=n, relu=True, res=True, scale=0.7)
    x, calls, bias, res, os_ = _setup(c, ci + co + T)
    batch = _run(c, x, calls, bias, res, os_, tc=True, route=route)
    one = Case(route, ci, co, T, [-3, 0, 3], n=1, relu=True, res=True, scale=0.7)
    alone = _run(one, x[4:5].contiguous(), calls, bias, res[4:5].contiguous(), os_, tc=True, route=route)
    torch.cuda.synchronize()
    assert torch.equal(batch[4:5], alone)


@pytest.mark.parametrize("T,n", [(5000, 6), (127, 300)])
@pytest.mark.parametrize("C_", [32, 64])
def test_tensor_core_resblock_clip_alone_equals_clip_in_batch(T, n, C_):
    w1, b1, w2, b2 = _block_weights(C_, C_, T)
    x = torch.randn(n, T, C_, device="cuda")
    batch = torch.empty_like(x)
    resblock_tc(x, batch, w1, b1, w2, b2, T, C_, 27, 0.7)
    xa = x[4:5].contiguous()
    alone = torch.empty_like(xa)
    resblock_tc(xa, alone, w1, b1, w2, b2, T, C_, 27, 0.7)
    torch.cuda.synchronize()
    assert torch.equal(batch[4:5], alone)


@pytest.mark.parametrize("route,ci,co,T,tc", [("narrow", 64, 1, 300, False), ("tile64", 64, 64, 300, False),
                                              ("tile32", 36, 32, 300, False), ("generic", 33, 48, 300, False),
                                              ("t5", 64, 32, 300, True), ("h2", 32, 64, 100, True)])
def test_phase_call_leaves_the_other_phase_untouched(route, ci, co, T, tc):
    """out_stride 2: each phase writes its own rows only; the other phase's rows keep the NaN they were filled with"""
    c = Case(route, ci, co, T, [1, 0], n=2, ostride=(2, 1), res=True, scale=0.7)
    x, calls, bias, res, os_ = _setup(c, T)
    out = _run(c, x, calls, bias, res, os_, tc=tc, route=route)
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[:, 0::2]).all()) and not bool(torch.isnan(out[:, 1::2]).any())
