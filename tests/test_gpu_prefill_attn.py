"""The chunked prefill's attention kernels (csrc/prefill.cu) against float64, at their tile edges, on every route.

jk_prefill_attention_f16 runs the per-layer attention of jk_prior_prefill: the forward output and the recorded weights of
one layer, on the tensor-core kernels (attn_fwd_mma_kernel / attn_record_mma_kernel, head tile DH 32 / 64 / 128 / 256
with 16-byte cp.async staging, DH 160 / 256 with 4-byte words) or the scalar kernels (attn_fwd_kernel /
attn_record_kernel: odd dh, dh > 256).  Every case runs on route 0 (the prefill's own choice, asserted against the
route the case was written for) and route 1 (the scalar kernels), forward and record in one call.

The reference is float64 over the reference's key sets (oracle.attn_layout_np.reference_keys; every encoder row for
attn_func 6), with the prefill's documented rounding points: s = fp16(fp32(fp16(q.k)) * scale2), softmax in fp64,
P.V in fp64.

Exact-score inputs: q and k are small integers / 4, so every product is a multiple of 2^-4 and every partial sum of the
<= 480 products stays far below 2^24 of those units.  q.k is then exact in any fp32 summation order (and on the tensor
cores, whose accumulation is expected, not measured, to be exact here), so the kernels' scores are the reference's
scores bitwise.  On these inputs:
  - recorded weights: |w - fp16(e_j / l)| <= one fp16 ulp of the reference (2^-24 among the subnormals), with
    e_j = exp(s_j - max s), l = sum e_j; every entry outside the pattern, and every row without keys, exactly 0;
  - forward output, per element, with u = 2^-11:
      |o - o_ref| <= 1.05 (sum_j max(u e_j, 2^-25) |v_jd| / l + u |o_ref|) + 1e-5 sum_j e_j |v_jd| / l
    the first term is the fp16 rounding of P (absolute 2^-25 below the fp16 normal range; the tensor-core kernel's
    running-max P is rescaled by exp(m_run - m) <= 1, so the same bound holds for it), the second the output rounding,
    the third an estimate for the fp32 exponentials, sums and rescales.  One key missing or extra among <= 500 moves an
    element by about |v - o| / nk, far outside this bound.
Realistic inputs (full-mantissa q, k) add a score-flip term: the kernel's fp32 q.k differs from the exact one by at most
gamma = dh 2^-24 of sum_d |q_d k_d|, and the two fp16 roundings by at most 2^-10 of |s| each, so
  ds_j <= 2^-9 |s_j| + scale2 gamma sum_d |q_d k_jd|,  |do| <= 1.05 sum_j (e_j / l) ds_j |v_jd - o_ref|,
  |dw_j| <= 1.05 w_j (ds_j + sum_i w_i ds_i)  (on top of the rounding bounds above).
Poisoning: K / V rows the pattern never reads (rows >= prime for attn_func 7, the last block for 3) and the cache columns
dh .. dh_pad of attn_func 6 hold fp16 NaN; out and w start as NaN, and a guard after each buffer must be unchanged."""
import ctypes as C
import math
import zlib
from dataclasses import dataclass

import pytest
import torch

from jukebox_b200 import _lib
from jukebox_b200._lib import lib, stream_ptr

pytestmark = pytest.mark.gpu

U = 2.0 ** -11
GUARD = 256                                  # fp16 elements after each output buffer
CHUNK_ELEMS = 1 << 25                        # float64 elements of one gathered [queries, keys, dh] block


# ---- the reference's key sets, vectorised --------------------------------------------------------------------------
def key_mask(attn_func, P, bc, prime, enc_rows=0, device="cpu"):
    """[P, keys] bool: key j of query p (positions < P; for attn_func 6 the encoder rows), reference_keys as a mask"""
    q = torch.arange(P, device=device)[:, None]
    if attn_func == 6:
        return torch.ones(P, enc_rows, dtype=torch.bool, device=device)
    k = torch.arange(P, device=device)[None, :]
    causal = k <= q
    if attn_func == 0:
        return causal
    if attn_func == 1:
        return causal & (k // bc == q // bc)
    if attn_func == 2:
        return causal & (k % bc == q % bc)
    if attn_func == 3:
        return k // bc == q // bc - 1
    if attn_func == 7:
        return causal & (k < prime)
    raise ValueError(attn_func)


def key_lists(mask):
    """mask [P, keys] -> idx [P, maxk] (key indices in increasing order, padded with 0), valid [P, maxk]"""
    cnt = mask.sum(1)
    maxk = max(int(cnt.max()), 1)
    order = torch.argsort((~mask).to(torch.int8), dim=1, stable=True)[:, :maxk]
    valid = torch.arange(maxk, device=mask.device)[None, :] < cnt[:, None]
    return torch.where(valid, order, torch.zeros_like(order)), valid


def exact_grid(shape, lim, generator, device="cpu"):
    """fp16 integers in [-lim, lim] / 4 (lim: a number or a tensor broadcast against shape): fp16-exact, and any dot
    product of <= 480 of them is exact in fp32"""
    u = torch.rand(shape, generator=generator, device=device, dtype=torch.float64)
    lim = torch.as_tensor(lim, device=device, dtype=torch.float64)
    return (torch.floor(u * (2 * lim + 1)) - lim).div(4).half()


def scale2_of(dh):
    """engine.cuh attn_scale2: (1 / sqrt(sqrt(dh)))^2 rounded to fp32"""
    sc = 1.0 / math.sqrt(math.sqrt(dh))
    return torch.tensor(sc * sc, dtype=torch.float32).item()


def fp16_ulp(x):
    """one fp16 ulp of fp16-representable x >= 0 (float64): 2^-24 below the normal range"""
    _, e = torch.frexp(x)
    return torch.where(x < 2.0 ** -14, torch.full_like(x, 2.0 ** -24), torch.ldexp(torch.ones_like(x), e - 11))


def reference(q, k, v, idx, valid, dh, exact):
    """one (sample, head): q [P, dh], k / v [keys, dh] fp16 -> float64 o_ref [P, dh], the forward bound [P, dh],
    w_ref [P, maxk] (e_j / l at the keys idx) and the record bound [P, maxk]"""
    P, maxk = idx.shape
    s2 = scale2_of(dh)
    o_ref = torch.zeros(P, dh, dtype=torch.float64, device=q.device)
    o_bnd = torch.zeros_like(o_ref)
    w_ref = torch.zeros(P, maxk, dtype=torch.float64, device=q.device)
    w_bnd = torch.zeros_like(w_ref)
    step = max(1, CHUNK_ELEMS // (maxk * dh))
    for p0 in range(0, P, step):
        sl = slice(p0, min(P, p0 + step))
        ok = valid[sl]
        kk, vv = k[idx[sl]].double(), v[idx[sl]].double()                 # [c, maxk, dh]
        qq = q[sl].double()
        dot = torch.einsum("pd,pkd->pk", qq, kk)
        s = (dot.half().float() * s2).half().double()
        s = torch.where(ok, s, torch.full_like(s, -math.inf))
        mx = s.max(1, keepdim=True).values
        mx = torch.where(torch.isfinite(mx), mx, torch.zeros_like(mx))
        e = torch.exp(s - mx)                                               # 0 outside the pattern
        l = e.sum(1, keepdim=True)
        inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
        w = e * inv
        o = torch.einsum("pk,pkd->pd", w, vv)
        av = vv.abs()
        pr = torch.where(ok, torch.clamp(U * e, min=2.0 ** -25), torch.zeros_like(e))
        bnd = 1.05 * (torch.einsum("pk,pkd->pd", pr, av) * inv + U * o.abs()) + 1e-5 * torch.einsum("pk,pkd->pd", w, av)
        wb = fp16_ulp(w.half().double())
        if not exact:
            gamma = dh * 2.0 ** -24
            ds = 2.0 ** -9 * torch.where(ok, s.abs(), torch.zeros_like(s)) + s2 * gamma * torch.einsum("pd,pkd->pk", qq.abs(), kk.abs())
            ds = torch.where(ok, ds, torch.zeros_like(ds))
            bnd = bnd + 1.05 * torch.einsum("pk,pkd->pd", w * ds, (vv - o[:, None, :]).abs())
            wb = wb + 1.05 * w * (ds + (w * ds).sum(1, keepdim=True))
        o_ref[sl], o_bnd[sl], w_ref[sl], w_bnd[sl] = o, bnd, w, torch.where(ok, wb, torch.zeros_like(wb))
    return o_ref, o_bnd, w_ref, w_bnd


# ---- cases --------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    attn_func: int
    dh: int
    P: int
    n: int = 1
    H: int = 2
    bc: int = 0
    prime: int = 0
    enc_rows: int = 0
    dh_pad: int = 0                  # 0: dh rounded up to 16, as the engine pads its caches
    ld: int = 0                      # 0: every key (P, or enc_rows)
    route: tuple = None              # (tile_dh, stage_bytes) route 0 takes; None: the scalar kernels
    exact: bool = True
    qmax: int = 24                   # q integers of a row lie in [-r, r], r drawn from 1 .. qmax per row (k: [-8, 8])

    def __post_init__(self):
        self.dh_pad = self.dh_pad or -(-self.dh // 16) * 16
        self.ld = self.ld or (self.enc_rows if self.attn_func == 6 else self.P)

    def __str__(self):
        return self.name


R32, R64, R128, R256, R160W4, R256W4 = (32, 16), (64, 16), (128, 16), (256, 16), (160, 4), (256, 4)
CASES = [
    *[Case(f"dh16-dense-P{P}", 0, 16, P, n=2, H=4, route=R32) for P in (1, 31, 33, 64, 65, 129)],
    Case("dh64-block-bc16-P61", 1, 64, 61, n=3, H=1, bc=16, route=R64),
    Case("dh64-transpose-bc16-P1100", 2, 64, 1100, n=1, H=2, bc=16, route=R64),
    Case("dh64-prevblock-bc65-P200", 3, 64, 200, n=2, H=2, bc=65, route=R64),
    *[Case(f"dh64-prime48-P{P}", 7, 64, P, n=2, H=1, prime=48, ld=40, route=R64) for P in (30, 48, 100)],
    Case("dh40-dense-P97", 0, 40, 97, n=1, H=4, route=R64),
    Case("dh80-dense-P512", 0, 80, 512, n=1, H=4, route=R128),
    Case("dh128-encdec-rows1", 6, 128, 130, n=2, H=1, enc_rows=1, route=R128),
    Case("dh128-encdec-rows33", 6, 128, 130, n=1, H=2, enc_rows=33, route=R128),
    Case("dh128-encdec-rows512-pad144", 6, 128, 130, n=2, H=2, enc_rows=512, dh_pad=144, route=R128),
    Case("dh256-dense-P4096", 0, 256, 4096, n=1, H=2, route=R256),
    Case("dh256-prime384-P800", 7, 256, 800, n=1, H=2, prime=384, ld=384, route=R256),
    Case("dh150-transpose-bc128-P8192", 2, 150, 8192, n=1, H=8, bc=128, route=R160W4),
    Case("dh150-block-bc128-P300", 1, 150, 300, n=2, H=1, bc=128, route=R160W4),
    Case("dh150-prevblock-bc128-P300", 3, 150, 300, n=1, H=2, bc=128, route=R160W4),
    Case("dh150-encdec-rows512", 6, 150, 100, n=1, H=4, enc_rows=512, route=R160W4),
    Case("dh170-dense-P70", 0, 170, 70, n=3, H=1, route=R256W4),
    Case("dh480-block-bc128-P300", 1, 480, 300, n=1, H=1, bc=128),
    Case("dh480-transpose-bc128-P2048", 2, 480, 2048, n=1, H=2, bc=128),
    Case("dh75-dense-P40", 0, 75, 40, n=2, H=2),
    Case("dh258-prevblock-bc32-P100", 3, 258, 100, n=1, H=2, bc=32),
    # full-mantissa q, k: one per route
    Case("real-dh16-dense-P129", 0, 16, 129, n=2, H=2, route=R32, exact=False),
    Case("real-dh64-prevblock-bc65-P200", 3, 64, 200, n=1, H=2, bc=65, route=R64, exact=False),
    Case("real-dh80-dense-P512", 0, 80, 512, n=1, H=1, route=R128, exact=False),
    Case("real-dh256-prime384-P500", 7, 256, 500, n=1, H=1, prime=384, route=R256, exact=False),
    Case("real-dh150-transpose-bc128-P1024", 2, 150, 1024, n=1, H=2, bc=128, route=R160W4, exact=False),
    Case("real-dh170-dense-P70", 0, 170, 70, n=1, H=2, route=R256W4, exact=False),
    Case("real-dh480-block-bc128-P300", 1, 480, 300, n=1, H=1, bc=128, exact=False),
]


def nan16(shape):
    return torch.full(shape, float("nan"), dtype=torch.float16, device="cuda")


def make_inputs(c, g):
    """qkv [n * P, q_stride] (+ caches for attn_func 6), with the rows and columns no kernel should read set to NaN"""
    S = c.H * c.dh
    enc = c.attn_func == 6
    nk_rows = c.enc_rows if enc else c.P

    def qk(shape, rows_lim):
        if c.exact:
            return exact_grid(shape, rows_lim, g, "cuda")
        return (torch.randn(shape, generator=g, device="cuda") * 1.5).half()

    rq = torch.randint(1, c.qmax + 1, (c.n, c.P, c.H, 1), generator=g, device="cuda")
    q = qk((c.n, c.P, c.H, c.dh), rq)
    k = qk((c.n, nk_rows, c.H, c.dh), 8)
    v = torch.randn((c.n, nk_rows, c.H, c.dh), generator=g, device="cuda").half()
    if enc:
        qkv = q.reshape(c.n * c.P, S).contiguous()
        kc, vc = nan16((c.n, c.H, c.enc_rows, c.dh_pad)), nan16((c.n, c.H, c.enc_rows, c.dh_pad))
        kc[..., :c.dh] = k.permute(0, 2, 1, 3)
        vc[..., :c.dh] = v.permute(0, 2, 1, 3)
        return qkv, kc, vc, q, k, v
    qkv = torch.cat([q.reshape(c.n, c.P, S), k.reshape(c.n, c.P, S), v.reshape(c.n, c.P, S)], 2)
    unread = torch.zeros(c.P, dtype=torch.bool, device="cuda")
    if c.attn_func == 7:
        unread[c.prime:] = True
    if c.attn_func == 3:
        unread[(-(-c.P // c.bc) - 1) * c.bc:] = True
    qkv[:, unread, S:] = float("nan")
    return qkv.reshape(c.n * c.P, 3 * S).contiguous(), None, None, q, k, v


def with_guard(numel, g):
    buf = nan16((numel + GUARD,))
    buf[numel:] = torch.randn(GUARD, generator=g, device="cuda").half()
    return buf, buf[numel:].clone()


def run_case(c, route):
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.name.encode()))
    qkv, kc, vc, q, k, v = make_inputs(c, g)
    S = c.H * c.dh
    out, out_guard = with_guard(c.n * c.P * S, g)
    w, w_guard = with_guard(c.n * c.H * c.P * c.ld, g)
    a = _lib.PrefillAttnArgs(qkv=qkv.data_ptr(), k_cache=kc.data_ptr() if kc is not None else None,
                             v_cache=vc.data_ptr() if vc is not None else None, out=out.data_ptr(), w=w.data_ptr(),
                             ld=c.ld, n=c.n, P=c.P, heads=c.H, dh=c.dh, dh_pad=c.dh_pad, attn_func=c.attn_func, bc=c.bc,
                             prime=c.prime, enc_rows=c.enc_rows, route=route)
    taken = _lib.PrefillAttnRoute()
    rc = lib().jk_prefill_attention_f16(C.byref(a), C.byref(taken), stream_ptr())
    assert rc == 0, lib().jk_last_error().decode()
    torch.cuda.synchronize()
    got = (taken.tensor_cores, taken.tile_dh, taken.stage_bytes)
    want = (1, *c.route) if route == 0 and c.route else (0, 0, 0)
    assert got == want, f"{c}: route {route} ran {got}, the case targets {want}"
    assert torch.equal(out[-GUARD:], out_guard), f"{c}: store past the end of out"
    assert torch.equal(w[-GUARD:], w_guard), f"{c}: store past the end of w"
    return out[:-GUARD].view(c.n, c.P, c.H, c.dh), w[:-GUARD].view(c.n, c.H, c.P, c.ld), q, k, v


def check_case(c, route):
    out, w, q, k, v = run_case(c, route)
    mask = key_mask(c.attn_func, c.P, c.bc, c.prime, c.enc_rows, "cuda")
    idx, valid = key_lists(mask)
    no_keys = ~mask.any(1)
    rec = valid & (idx < c.ld)
    worst_o = worst_w = 0.0
    for b in range(c.n):
        for h in range(c.H):
            o_ref, o_bnd, w_ref, w_bnd = reference(q[b, :, h], k[b, :, h], v[b, :, h], idx, valid, c.dh, c.exact)
            o = out[b, :, h].double()
            assert not torch.isnan(o).any(), f"{c} b{b} h{h}: NaN in the output (unwritten, or a poisoned read)"
            assert (o[no_keys] == 0).all(), f"{c} b{b} h{h}: a row without keys is not 0"
            err = (o - o_ref).abs()
            bad = err > o_bnd
            if bad.any():
                p, d = [int(t) for t in bad.nonzero()[0]]
                pytest.fail(f"{c} route {route} b{b} h{h}: {int(bad.sum())} output elements out of bound, first p {p} "
                            f"d {d}: {o[p, d].item()} vs {o_ref[p, d].item()} (bound {o_bnd[p, d].item():.3g})")
            worst_o = max(worst_o, float((err / o_bnd.clamp_min(1e-30)).max()))
            wk = w[b, h]
            rows = torch.arange(c.P, device="cuda")[:, None].expand_as(idx)
            wg = wk[rows[rec], idx[rec]].double()
            werr = (wg - w_ref[rec].half().double()).abs() if c.exact else (wg - w_ref[rec]).abs()
            wbad = werr > w_bnd[rec]
            if wbad.any():
                i = int(wbad.nonzero()[0])
                pytest.fail(f"{c} route {route} b{b} h{h}: {int(wbad.sum())} recorded weights out of bound, query "
                            f"{int(rows[rec][i])} key {int(idx[rec][i])}: {wg[i].item()} vs {w_ref[rec][i].item()}")
            worst_w = max(worst_w, float((werr / w_bnd[rec]).max()) if rec.any() else 0.0)
            rest = wk.clone()
            rest[rows[rec], idx[rec]] = 0
            assert (rest == 0).all(), f"{c} route {route} b{b} h{h}: recorded weight outside the pattern (or not zeroed)"
    print(f"{c} route {route}: worst output error {worst_o:.3f} of its bound, weights {worst_w:.3f}")


@pytest.mark.parametrize("route", [0, 1])
@pytest.mark.parametrize("case", CASES, ids=str)
def test_prefill_attention_against_float64(case, route):
    check_case(case, route)
