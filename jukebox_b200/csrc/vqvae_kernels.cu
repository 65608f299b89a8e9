// VQ-VAE kernels (fp32, channels-last [N, T, C]) and small fp32 helpers used once per window.
//
// Reference (under /root/reference/jukebox/vqvae/): bottleneck.py:112-123 (quantise / dequantise),
// encdec.py:6-131 and resnet.py:27-75 (Conv1d / ConvTranspose1d / ResConv1DBlock stacks).
// The encoder feeds an argmin whose indices must be bit-exact, so these kernels keep true fp32 FMA
// arithmetic (no TF32): see DESIGN.md "VQ-VAE numerics".
#include "split_tma.cuh"
#include <algorithm>
#include "../../include/jkb200.h"

using namespace jk;

namespace {

// ---------------------------------------------------------------------------------------
// codebook argmin.  64 rows per CTA, x rows live in registers, the codebook streams through
// shared memory in tiles of 128 codes; the distance matrix is never materialised.
// dist = (|x|^2 - 2 x.k) + |k|^2 evaluated in fp32 exactly as bottleneck.py:115-117 associates it.
// ---------------------------------------------------------------------------------------
template <int WIDTH>
__global__ void __launch_bounds__(256) vq_argmin_kernel(const float* __restrict__ x, const float* __restrict__ cb,
                                                        long long* __restrict__ idx, float* __restrict__ mind,
                                                        long long n, int kbins) {
    constexpr int TILE = 128;
    __shared__ __align__(16) float cs[TILE][WIDTH];
    __shared__ float kk[TILE];
    __shared__ float bd[4][64];
    __shared__ int bi[4][64];
    const int tid = threadIdx.x, r = tid & 63, q = tid >> 6;
    const long long row = (long long)blockIdx.x * 64 + r;
    float xr[WIDTH];
    float xx = 0.f;
    if (row < n) {
#pragma unroll
        for (int d = 0; d < WIDTH; d += 4) {
            float4 v = *reinterpret_cast<const float4*>(x + row * WIDTH + d);
            xr[d] = v.x; xr[d + 1] = v.y; xr[d + 2] = v.z; xr[d + 3] = v.w;
        }
#pragma unroll
        for (int d = 0; d < WIDTH; ++d) xx += xr[d] * xr[d];
    } else {
#pragma unroll
        for (int d = 0; d < WIDTH; ++d) xr[d] = 0.f;
    }
    float best = INFINITY;
    int besti = 0;
    for (int c0 = 0; c0 < kbins; c0 += TILE) {
        __syncthreads();
        for (int i = tid; i < TILE * WIDTH / 4; i += 256) {
            int j = i / (WIDTH / 4), d4 = i % (WIDTH / 4);
            float4 v = make_float4(0, 0, 0, 0);
            if (c0 + j < kbins) v = *reinterpret_cast<const float4*>(cb + (size_t)(c0 + j) * WIDTH + d4 * 4);
            *reinterpret_cast<float4*>(&cs[j][d4 * 4]) = v;
        }
        __syncthreads();
        if (tid < TILE) {
            float s = 0.f;
#pragma unroll
            for (int d = 0; d < WIDTH; ++d) s += cs[tid][d] * cs[tid][d];
            kk[tid] = s;
        }
        __syncthreads();
        const int jend = min(TILE, kbins - c0);
        for (int j = q * (TILE / 4); j < (q + 1) * (TILE / 4) && j < jend; ++j) {
            float dot = 0.f;
#pragma unroll
            for (int d = 0; d < WIDTH; d += 4) {
                float4 k4 = *reinterpret_cast<const float4*>(&cs[j][d]);
                dot = fmaf(xr[d], k4.x, dot);
                dot = fmaf(xr[d + 1], k4.y, dot);
                dot = fmaf(xr[d + 2], k4.z, dot);
                dot = fmaf(xr[d + 3], k4.w, dot);
            }
            float dist = (xx - 2.0f * dot) + kk[j];
            if (dist < best) { best = dist; besti = c0 + j; }
        }
    }
    bd[q][r] = best;
    bi[q][r] = besti;
    __syncthreads();
    if (q == 0 && row < n) {
        float b = bd[0][r];
        int bidx = bi[0][r];
#pragma unroll
        for (int qq = 1; qq < 4; ++qq) {
            float d = bd[qq][r];
            int i = bi[qq][r];
            if (d < b || (d == b && i < bidx)) { b = d; bidx = i; }
        }
        idx[row] = bidx;
        if (mind) mind[row] = b;
    }
}

// generic width (multiple of 4, <= 512): one warp per row, lanes over codes
__global__ void vq_argmin_generic_kernel(const float* __restrict__ x, const float* __restrict__ cb,
                                         long long* __restrict__ idx, float* __restrict__ mind, long long n, int kbins,
                                         int width) {
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    const float* xr = x + row * width;
    float xx = 0.f;
    for (int d = 0; d < width; ++d) xx += xr[d] * xr[d];
    float best = INFINITY;
    int besti = 0x7fffffff;
    for (int j = lane; j < kbins; j += 32) {
        const float* k = cb + (size_t)j * width;
        float dot = 0.f, ks = 0.f;
        for (int d = 0; d < width; ++d) { dot = fmaf(xr[d], k[d], dot); ks += k[d] * k[d]; }
        float dist = (xx - 2.0f * dot) + ks;
        if (dist < best) { best = dist; besti = j; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        float ob = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (ob < best || (ob == best && oi < besti)) { best = ob; besti = oi; }
    }
    if (lane == 0) { idx[row] = besti; if (mind) mind[row] = best; }
}

__global__ void vq_gather_kernel(const long long* __restrict__ idx, const float* __restrict__ cb, float* __restrict__ out,
                                 long long n, int kbins, int width4) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * width4) return;
    const long long r = i / width4;
    const int d = (int)(i % width4);
    long long j = idx[r];
    j = j < 0 ? 0 : (j >= kbins ? kbins - 1 : j);
    reinterpret_cast<float4*>(out)[i] = reinterpret_cast<const float4*>(cb)[j * width4 + d];
}

// ---------------------------------------------------------------------------------------
// generic channels-last conv: tile of 64 positions x 64 output channels per CTA,
// K = taps x c_in walked in slabs of 32 input channels through shared memory.
// ---------------------------------------------------------------------------------------
struct ConvP {
    const float* in; long long t_in; int c_in;
    float* out; long long t_out; int c_out;
    const float* w; const float* bias; const float* res;
    int n_taps; int tap_off[4]; int in_stride; int out_stride; int out_offset; int relu_in; float scale;
};

__global__ void __launch_bounds__(256) conv1d_cl_kernel(ConvP P) {
    constexpr int TT = 64, CT = 64, KC = 32;
    __shared__ float xs[KC][TT + 1];
    __shared__ __align__(16) float ws[KC][CT];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const long long t0 = (long long)blockIdx.x * TT;
    const int co0 = blockIdx.y * CT;
    const int nb = blockIdx.z;
    const float* in = P.in + (size_t)nb * P.t_in * P.c_in;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int tap = 0; tap < P.n_taps; ++tap) {
        const int off = P.tap_off[tap];
        for (int ci0 = 0; ci0 < P.c_in; ci0 += KC) {
            __syncthreads();
            for (int i = tid; i < KC * TT; i += 256) {
                const int k = i % KC, tt = i / KC;
                const long long tp = (t0 + tt) * P.in_stride + off;
                float v = 0.f;
                if (ci0 + k < P.c_in && tp >= 0 && tp < P.t_in && t0 + tt < P.t_out) {
                    v = in[(size_t)tp * P.c_in + ci0 + k];
                    if (P.relu_in) v = fmaxf(v, 0.f);
                }
                xs[k][tt] = v;
            }
            for (int i = tid; i < KC * CT; i += 256) {
                const int c = i % CT, k = i / CT;
                float v = 0.f;
                if (ci0 + k < P.c_in && co0 + c < P.c_out) v = P.w[((size_t)tap * P.c_in + ci0 + k) * P.c_out + co0 + c];
                ws[k][c] = v;
            }
            __syncthreads();
#pragma unroll 8
            for (int k = 0; k < KC; ++k) {
                float a[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) a[i] = xs[k][ty * 4 + i];
                const float4 b = *reinterpret_cast<const float4*>(&ws[k][tx * 4]);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    acc[i][0] = fmaf(a[i], b.x, acc[i][0]);
                    acc[i][1] = fmaf(a[i], b.y, acc[i][1]);
                    acc[i][2] = fmaf(a[i], b.z, acc[i][2]);
                    acc[i][3] = fmaf(a[i], b.w, acc[i][3]);
                }
            }
        }
    }
    const long long rows_out = P.t_out * P.out_stride;
    float* out = P.out + (size_t)nb * rows_out * P.c_out;
    const float* res = P.res ? P.res + (size_t)nb * rows_out * P.c_out : nullptr;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long t = t0 + ty * 4 + i;
        if (t >= P.t_out) continue;
        const long long orow = t * P.out_stride + P.out_offset;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int co = co0 + tx * 4 + j;
            if (co >= P.c_out) continue;
            float v = P.scale * (acc[i][j] + (P.bias ? P.bias[co] : 0.f));
            if (res) v += res[(size_t)orow * P.c_out + co];
            out[(size_t)orow * P.c_out + co] = v;
        }
    }
}

// ---------------------------------------------------------------------------------------
// Fused ResConv1DBlock (resnet.py:27-44) for the VQ-VAE's own shapes (n_in == n_state == C, C = 32 or 64):
//   out = x + res_scale * (W2 . relu(W1 (*) relu(x) + b1) + b2),   W1: 3 taps with dilation d, W2: 1 x 1
// One CTA = one tile of TT positions of one clip.  Both weight matrices, the three (relu'd) input tap tiles and
// the hidden tile live in shared memory; the hidden activation never goes to HBM (the two-launch form wrote
// and re-read it: 2 x 4 x C bytes per position of 5 x 4 x C).  Each thread owns 8 positions x 4 channels; per
// 4 k-steps it issues 8 + 4 LDS.128 for 128 FMAs (the generic kernel: 20 LDS for 64), with the position
// mapping (ty + TY * i) chosen so that the lanes of a warp read at most TX-strided rows 1 apart: no bank
// conflicts with the 4-float row padding.  fp32 FMAs in the generic kernel's order (tap, then input channel), so both
// paths agree to the last bit on everything before the residual add; the add itself is rounded differently (the two
// agree bitwise for a power-of-two res_scale, and within one rounding of x + res_scale * y otherwise).
// ---------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256, 1)
resblock_fused_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ w1,
                      const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                      long long T, int dil, float rs) {
    constexpr int TX = C / 4, TY = 256 / TX, TT = TY * 8, XS = C + 4;
    extern __shared__ __align__(16) float rsm[];
    float* w1s = rsm;                    // [3][C][C]
    float* w2s = w1s + 3 * C * C;        // [C][C]
    float* xs = w2s + C * C;             // [3][TT][XS]  relu(x) at t + (tap - 1) * dil
    float* hs = xs + 3 * TT * XS;        // [TT][XS]     relu(hidden)
    const int tid = threadIdx.x, tx = tid % TX, ty = tid / TX;
    const long long t0 = (long long)blockIdx.x * TT;
    const float* xin = x + (size_t)blockIdx.y * T * C;
    float* xout = out + (size_t)blockIdx.y * T * C;
    for (int i = tid; i < 3 * C * C / 4; i += 256) reinterpret_cast<float4*>(w1s)[i] = __ldg(reinterpret_cast<const float4*>(w1) + i);
    for (int i = tid; i < C * C / 4; i += 256) reinterpret_cast<float4*>(w2s)[i] = __ldg(reinterpret_cast<const float4*>(w2) + i);
#pragma unroll
    for (int tap = 0; tap < 3; ++tap) {
        const long long off = (long long)(tap - 1) * dil;
#pragma unroll 4
        for (int i = tid; i < TT * TX; i += 256) {
            const int t = i / TX, c4 = i % TX;
            const long long tp = t0 + t + off;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tp >= 0 && tp < T) v = __ldg(reinterpret_cast<const float4*>(xin + (size_t)tp * C) + c4);
            v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
            *reinterpret_cast<float4*>(xs + ((size_t)tap * TT + t) * XS + c4 * 4) = v;
        }
    }
    __syncthreads();
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#define JK_RB_STEP(XBASE, WBASE)                                                                  \
    {                                                                                             \
        const float4 wa = *reinterpret_cast<const float4*>((WBASE) + 0 * C + tx * 4);             \
        const float4 wb = *reinterpret_cast<const float4*>((WBASE) + 1 * C + tx * 4);             \
        const float4 wc = *reinterpret_cast<const float4*>((WBASE) + 2 * C + tx * 4);             \
        const float4 wd = *reinterpret_cast<const float4*>((WBASE) + 3 * C + tx * 4);             \
        _Pragma("unroll") for (int i = 0; i < 8; ++i) {                                           \
            const float4 xv = *reinterpret_cast<const float4*>((XBASE) + (size_t)(ty + TY * i) * XS); \
            acc[i][0] = fmaf(xv.x, wa.x, acc[i][0]); acc[i][1] = fmaf(xv.x, wa.y, acc[i][1]);      \
            acc[i][2] = fmaf(xv.x, wa.z, acc[i][2]); acc[i][3] = fmaf(xv.x, wa.w, acc[i][3]);      \
            acc[i][0] = fmaf(xv.y, wb.x, acc[i][0]); acc[i][1] = fmaf(xv.y, wb.y, acc[i][1]);      \
            acc[i][2] = fmaf(xv.y, wb.z, acc[i][2]); acc[i][3] = fmaf(xv.y, wb.w, acc[i][3]);      \
            acc[i][0] = fmaf(xv.z, wc.x, acc[i][0]); acc[i][1] = fmaf(xv.z, wc.y, acc[i][1]);      \
            acc[i][2] = fmaf(xv.z, wc.z, acc[i][2]); acc[i][3] = fmaf(xv.z, wc.w, acc[i][3]);      \
            acc[i][0] = fmaf(xv.w, wd.x, acc[i][0]); acc[i][1] = fmaf(xv.w, wd.y, acc[i][1]);      \
            acc[i][2] = fmaf(xv.w, wd.z, acc[i][2]); acc[i][3] = fmaf(xv.w, wd.w, acc[i][3]);      \
        }                                                                                         \
    }
#pragma unroll 1
    for (int tap = 0; tap < 3; ++tap) {
#pragma unroll 2
        for (int k4 = 0; k4 < C / 4; ++k4)
            JK_RB_STEP(xs + (size_t)tap * TT * XS + k4 * 4, w1s + ((size_t)tap * C + k4 * 4) * C)
    }
    {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(b1) + tx);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float4 h;
            h.x = fmaxf(acc[i][0] + bv.x, 0.f); h.y = fmaxf(acc[i][1] + bv.y, 0.f);
            h.z = fmaxf(acc[i][2] + bv.z, 0.f); h.w = fmaxf(acc[i][3] + bv.w, 0.f);
            *reinterpret_cast<float4*>(hs + (size_t)(ty + TY * i) * XS + tx * 4) = h;
            acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
        }
    }
    __syncthreads();
#pragma unroll 2
    for (int k4 = 0; k4 < C / 4; ++k4) JK_RB_STEP(hs + k4 * 4, w2s + (size_t)(k4 * 4) * C)
#undef JK_RB_STEP
    {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(b2) + tx);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const long long t = t0 + ty + TY * i;
            if (t >= T) continue;
            const float4 r = __ldg(reinterpret_cast<const float4*>(xin + (size_t)t * C) + tx);
            float4 v;
            v.x = rs * (acc[i][0] + bv.x); v.x += r.x;
            v.y = rs * (acc[i][1] + bv.y); v.y += r.y;
            v.z = rs * (acc[i][2] + bv.z); v.z += r.z;
            v.w = rs * (acc[i][3] + bv.w); v.w += r.w;
            *(reinterpret_cast<float4*>(xout + (size_t)t * C) + tx) = v;
        }
    }
}

// ---------------------------------------------------------------------------------------
// Tile conv for the VQ-VAE's wide layers (c_out = 32 or 64, c_in <= 64): the register tiling of the fused
// ResConv1DBlock kernel applied to one convolution - all taps' weights and (ReLU'd) input tap tiles in shared
// memory, 8 positions x 4 channels per thread, FMAs in the generic kernel's order (tap, then input channel),
// so results are bit-identical to conv1d_cl_kernel.  Covers the k4-s2 down / (two-phase) up-sampling convs and
// the k3 input convs, i.e. everything between the resblocks.
// ---------------------------------------------------------------------------------------
template <int CO>
__global__ void __launch_bounds__(256, 1) conv1d_cl_tile_kernel(ConvP P) {
    constexpr int TX = CO / 4, TY = 256 / TX, TT = TY * 8;
    extern __shared__ __align__(16) float csm[];
    const int CI = P.c_in, XS = CI + 4, NT = P.n_taps;
    float* ws = csm;                                   // [NT][CI][CO]
    float* xs = ws + (size_t)NT * CI * CO;             // [NT][TT][XS]
    const int tid = threadIdx.x, tx = tid % TX, ty = tid / TX;
    const long long t0 = (long long)blockIdx.x * TT;
    const float* in = P.in + (size_t)blockIdx.y * P.t_in * CI;
    for (int i = tid; i < NT * CI * CO / 4; i += 256) reinterpret_cast<float4*>(ws)[i] = __ldg(reinterpret_cast<const float4*>(P.w) + i);
    const int c4n = CI / 4;
    for (int tap = 0; tap < NT; ++tap) {
        const long long off = tap == 0 ? P.tap_off[0] : tap == 1 ? P.tap_off[1] : tap == 2 ? P.tap_off[2] : P.tap_off[3];
#pragma unroll 4
        for (int i = tid; i < TT * c4n; i += 256) {
            const int t = i / c4n, c4 = i - t * c4n;
            const long long tp = (t0 + t) * P.in_stride + off;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tp >= 0 && tp < P.t_in && t0 + t < P.t_out) v = __ldg(reinterpret_cast<const float4*>(in + (size_t)tp * CI) + c4);
            if (P.relu_in) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            *reinterpret_cast<float4*>(xs + ((size_t)tap * TT + t) * XS + c4 * 4) = v;
        }
    }
    __syncthreads();
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 1
    for (int tap = 0; tap < NT; ++tap) {
        const float* xb = xs + (size_t)tap * TT * XS;
        const float* wb = ws + (size_t)tap * CI * CO + tx * 4;
#pragma unroll 2
        for (int k4 = 0; k4 < c4n; ++k4) {
            const float4 wa = *reinterpret_cast<const float4*>(wb + (size_t)(k4 * 4 + 0) * CO);
            const float4 wq = *reinterpret_cast<const float4*>(wb + (size_t)(k4 * 4 + 1) * CO);
            const float4 wc = *reinterpret_cast<const float4*>(wb + (size_t)(k4 * 4 + 2) * CO);
            const float4 wd = *reinterpret_cast<const float4*>(wb + (size_t)(k4 * 4 + 3) * CO);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 xv = *reinterpret_cast<const float4*>(xb + (size_t)(ty + TY * i) * XS + k4 * 4);
                acc[i][0] = fmaf(xv.x, wa.x, acc[i][0]); acc[i][1] = fmaf(xv.x, wa.y, acc[i][1]);
                acc[i][2] = fmaf(xv.x, wa.z, acc[i][2]); acc[i][3] = fmaf(xv.x, wa.w, acc[i][3]);
                acc[i][0] = fmaf(xv.y, wq.x, acc[i][0]); acc[i][1] = fmaf(xv.y, wq.y, acc[i][1]);
                acc[i][2] = fmaf(xv.y, wq.z, acc[i][2]); acc[i][3] = fmaf(xv.y, wq.w, acc[i][3]);
                acc[i][0] = fmaf(xv.z, wc.x, acc[i][0]); acc[i][1] = fmaf(xv.z, wc.y, acc[i][1]);
                acc[i][2] = fmaf(xv.z, wc.z, acc[i][2]); acc[i][3] = fmaf(xv.z, wc.w, acc[i][3]);
                acc[i][0] = fmaf(xv.w, wd.x, acc[i][0]); acc[i][1] = fmaf(xv.w, wd.y, acc[i][1]);
                acc[i][2] = fmaf(xv.w, wd.z, acc[i][2]); acc[i][3] = fmaf(xv.w, wd.w, acc[i][3]);
            }
        }
    }
    const long long rows_out = P.t_out * P.out_stride;
    float* out = P.out + (size_t)blockIdx.y * rows_out * CO;
    const float* res = P.res ? P.res + (size_t)blockIdx.y * rows_out * CO : nullptr;
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (P.bias) bv = __ldg(reinterpret_cast<const float4*>(P.bias) + tx);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const long long t = t0 + ty + TY * i;
        if (t >= P.t_out) continue;
        const long long orow = t * P.out_stride + P.out_offset;
        float4 v;
        v.x = P.scale * (acc[i][0] + bv.x); v.y = P.scale * (acc[i][1] + bv.y);
        v.z = P.scale * (acc[i][2] + bv.z); v.w = P.scale * (acc[i][3] + bv.w);
        if (res) {
            const float4 r = __ldg(reinterpret_cast<const float4*>(res + (size_t)orow * CO) + tx);
            v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
        }
        *(reinterpret_cast<float4*>(out + (size_t)orow * CO) + tx) = v;
    }
}

template <int CO>
int launch_conv_tile(const ConvP& P, int n, cudaStream_t stream, bool* took) {
    constexpr int TX = CO / 4, TY = 256 / TX, TT = TY * 8;
    const size_t smem = ((size_t)P.n_taps * P.c_in * CO + (size_t)P.n_taps * TT * (P.c_in + 4)) * sizeof(float);
    *took = false;
    if (smem > 220 * 1024) return 0;
    if (int rc = set_max_smem_once<conv1d_cl_tile_kernel<CO>>(220 * 1024)) return rc;
    dim3 grid((unsigned)((P.t_out + TT - 1) / TT), (unsigned)n);
    conv1d_cl_tile_kernel<CO><<<grid, 256, smem, stream>>>(P);
    JK_CHECK_CUDA(cudaGetLastError());
    *took = true;
    return 0;
}

template <int C>
int launch_resblock_fused(const float* x, float* out, const float* w1, const float* b1, const float* w2, const float* b2,
                          int n, long long T, int dil, float rs, cudaStream_t stream) {
    constexpr int TX = C / 4, TY = 256 / TX, TT = TY * 8, XS = C + 4;
    constexpr size_t smem = (size_t)(4 * C * C + 4 * TT * XS) * sizeof(float);
    if (int rc = set_max_smem_once<resblock_fused_kernel<C>>((int)smem)) return rc;
    dim3 grid((unsigned)((T + TT - 1) / TT), (unsigned)n);
    resblock_fused_kernel<C><<<grid, 256, smem, stream>>>(x, out, w1, b1, w2, b2, T, dil, rs);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------
// ResConv1DBlock on the tensor cores, for the DECODER side (Decoder / Conditioner stacks: their outputs are audio and
// conditioning, never an argmin input, so summation order is free; the encoder keeps the exact-FMA kernel above).  This
// kernel takes the clips under 128 positions, which resblock_t5_kernel (vqvae_t5.cu) does not; like it, it needs 16-byte
// aligned x / out (and 8-byte aligned b1 / b2), which jk_resblock_tc checks.
// The fp16 x 3 split of split_tma.cuh on mma.sync.m16n8k16: x = hi + lo with hi = fp16(x), lo = fp16(x - hi): 22 mantissa
// bits, the same as a 3xTF32 split (fp16 and TF32 both carry 11 significant bits), products hi.w_hi + lo.w_hi + hi.w_lo
// accumulated in fp32.  Against 3xTF32 on m16n8k8: an MMA covers k = 16 instead of 8 at the same issue cost, operands are
// half the shared-memory bytes and arrive as whole fragments through ldmatrix (A: [position][channel] rows, B: [k][n] rows
// with .trans) - 10 ldmatrix + 24 MMA per k16 step at C = 64 where a TF32 kernel issued 32 LDS + 24 cvt/sub + 24 MMA for
// the same k range.  Values beyond the fp16 range saturate (cvt.satfinite); VQ-VAE activations are O(1).  Small
// activations lose nothing that matters: an fp16 remainder below 2^-14 is kept to an ABSOLUTE 2^-25.
//   * ONE WARP PER 16-POSITION TILE: a warp's output rows need only its own rows of the three tap tiles and of the hidden
//     tile, so nothing is shared between warps except the weights - no CTA barrier in the tile loop, and the sixteen warps
//     of a CTA (4 per scheduler) drift apart so that one's global loads overlap another's MMAs
//   * persistent CTAs (grid = #SMs), W1 / W2 hi + lo planes staged once per CTA
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"((uint32_t)__cvta_generic_to_shared(p)));
}

template <int C>
struct ResH2 {
    static constexpr int XS = C + 8;                       // halfs per row: 16-byte aligned rows an odd number of 16-byte units apart
    static constexpr int NT = C / 8, WARPS = 16;
    static constexpr int w_halfs = 2 * (3 * C + C) * XS;   // W1 hi, W1 lo, W2 hi, W2 lo
    static constexpr int warp_halfs = 2 * 16 * XS;         // ONE tap tile of a warp (hi, lo); the hidden tile reuses it
    static constexpr size_t smem = (size_t)(w_halfs + WARPS * warp_halfs) * 2;
};

// acc[nt] += A(16 x 16 at `ah`/`al`) . B(16 x C at `bh`/`bl`), three products of the split
template <int C>
__device__ __forceinline__ void h2_kstep(float (&acc)[C / 8][4], const __half* ah, const __half* al, const __half* bh, const __half* bl,
                                         int lane) {
    constexpr int XS = ResH2<C>::XS;
    const int r = lane & 15, c8 = (lane >> 4) * 8;
    uint32_t fh[4], fl[4];
    ldmatrix_x4(fh, ah + r * XS + c8);
    ldmatrix_x4(fl, al + r * XS + c8);
#pragma unroll
    for (int np = 0; np < C / 16; ++np) {
        uint32_t wh[4], wl[4];
        ldsm_x4_t(wh, bh + r * XS + np * 16 + c8);
        ldsm_x4_t(wl, bl + r * XS + np * 16 + c8);
        mma_16816(acc[2 * np], fl, wh[0], wh[1]);
        mma_16816(acc[2 * np], fh, wl[0], wl[1]);
        mma_16816(acc[2 * np], fh, wh[0], wh[1]);
        mma_16816(acc[2 * np + 1], fl, wh[2], wh[3]);
        mma_16816(acc[2 * np + 1], fh, wl[2], wl[3]);
        mma_16816(acc[2 * np + 1], fh, wh[2], wh[3]);
    }
}

// 16 warps per CTA (4 per scheduler; <= 128 registers each): a warp stages ONE tap tile at a time - the global loads of the
// next tap (or of the next tile's first tap) are in flight while the current tap's MMAs issue
template <int C>
__global__ void __launch_bounds__(512, 1)
resblock_h2_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ w1,
                   const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                   long long T, int dil, float rs, long long tiles_per_clip, long long total_tiles) {
    constexpr int XS = ResH2<C>::XS, NT = ResH2<C>::NT, WARPS = ResH2<C>::WARPS;
    extern __shared__ __align__(16) __half hsm[];
    __half* w1h = hsm;                          // [3 C][XS]
    __half* w1l = w1h + 3 * C * XS;
    __half* w2h = w1l + 3 * C * XS;             // [C][XS]
    __half* w2l = w2h + C * XS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __half* xh = w2l + C * XS + warp * ResH2<C>::warp_halfs;      // [16][XS] relu(x) at t + (tap - 1) * dil, then the hidden tile
    __half* xl = xh + 16 * XS;
    const int g = lane >> 2, t4 = lane & 3;
    for (int i = tid; i < 3 * C * C; i += WARPS * 32) {
        const int o = (i / C) * XS + i % C;
        split_f16(kWScale * __ldg(w1 + i), w1h[o], w1l[o]);
    }
    for (int i = tid; i < C * C; i += WARPS * 32) {
        const int o = (i / C) * XS + i % C;
        split_f16(kWScale * __ldg(w2 + i), w2h[o], w2l[o]);
    }
    __syncthreads();
    constexpr int TX = C / 4, PER = 16 * TX / 32, RJ = 32 / TX;   // float4 loads per lane per tap tile; rows between them
    const int lr = lane / TX, lc = lane % TX;             // this lane's row (+ j * RJ) and 16-byte chunk of a tap tile
    const long long stride = (long long)gridDim.x * WARPS;
    float4 v[PER];
    auto issue = [&](long long tile, int tap) {           // tap tile rows -> registers (zeros outside the clip)
        if (tile >= total_tiles) return;
        const long long nb = tile / tiles_per_clip;
        const long long tb = (tile - nb * tiles_per_clip) * 16 + (long long)(tap - 1) * dil + lr;
        const float4* p = reinterpret_cast<const float4*>(x + ((size_t)nb * T + tb) * C) + lc;
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            const long long tp = tb + j * RJ;
            v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tp >= 0 && tp < T) v[j] = __ldg(p + j * RJ * TX);
        }
    };
    long long tile = (long long)blockIdx.x * WARPS + warp;
    issue(tile, 0);
#pragma unroll 1
    for (; tile < total_tiles; tile += stride) {
        const long long nb = tile / tiles_per_clip, t0 = (tile - nb * tiles_per_clip) * 16;
        const float* xin = x + (size_t)nb * T * C;
        float* xout = out + (size_t)nb * T * C;
        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
        for (int tap = 0; tap < 3; ++tap) {
            __syncwarp();                       // the previous fragment reads of this buffer are done
#pragma unroll
            for (int j = 0; j < PER; ++j) {
                uint2 h, l;
                split_f16x2(fmaxf(v[j].x, 0.f), fmaxf(v[j].y, 0.f), h.x, l.x);
                split_f16x2(fmaxf(v[j].z, 0.f), fmaxf(v[j].w, 0.f), h.y, l.y);
                *reinterpret_cast<uint2*>(xh + (lr + j * RJ) * XS + lc * 4) = h;
                *reinterpret_cast<uint2*>(xl + (lr + j * RJ) * XS + lc * 4) = l;
            }
            if (tap < 2) issue(tile, tap + 1); else issue(tile + stride, 0);      // in flight during the MMAs below
            __syncwarp();
#pragma unroll
            for (int k16 = 0; k16 < C / 16; ++k16)
                h2_kstep<C>(acc, xh + k16 * 16, xl + k16 * 16, w1h + (tap * C + k16 * 16) * XS, w1l + (tap * C + k16 * 16) * XS, lane);
        }
        __syncwarp();                           // the tap tile is dead: the hidden tile takes its place
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {       // hidden = relu(conv1 + b1), split, -> shared memory (this warp's rows only)
            const int col = nt * 8 + 2 * t4;
            const float2 bv = __ldg(reinterpret_cast<const float2*>(b1 + col));
            uint32_t h, l;
            split_f16x2(fmaxf(fmaf(acc[nt][0], kWInv, bv.x), 0.f), fmaxf(fmaf(acc[nt][1], kWInv, bv.y), 0.f), h, l);
            *reinterpret_cast<uint32_t*>(xh + g * XS + col) = h;
            *reinterpret_cast<uint32_t*>(xl + g * XS + col) = l;
            split_f16x2(fmaxf(fmaf(acc[nt][2], kWInv, bv.x), 0.f), fmaxf(fmaf(acc[nt][3], kWInv, bv.y), 0.f), h, l);
            *reinterpret_cast<uint32_t*>(xh + (g + 8) * XS + col) = h;
            *reinterpret_cast<uint32_t*>(xl + (g + 8) * XS + col) = l;
            acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
        }
        __syncwarp();
#pragma unroll
        for (int k16 = 0; k16 < C / 16; ++k16)
            h2_kstep<C>(acc, xh + k16 * 16, xl + k16 * 16, w2h + k16 * 16 * XS, w2l + k16 * 16 * XS, lane);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {       // out = x + res_scale * (conv2 + b2): x exact from global memory
            const int col = nt * 8 + 2 * t4;
            const float2 bv = __ldg(reinterpret_cast<const float2*>(b2 + col));
#pragma unroll
            for (int hlf = 0; hlf < 2; ++hlf) {
                const long long t = t0 + g + 8 * hlf;
                if (t < T) {
                    const float2 r = __ldg(reinterpret_cast<const float2*>(xin + (size_t)t * C + col));
                    float2 o;
                    o.x = rs * fmaf(acc[nt][2 * hlf], kWInv, bv.x); o.x += r.x;
                    o.y = rs * fmaf(acc[nt][2 * hlf + 1], kWInv, bv.y); o.y += r.y;
                    *reinterpret_cast<float2*>(xout + (size_t)t * C + col) = o;
                }
            }
        }
    }
}

template <int C>
int launch_resblock_h2(const float* x, float* out, const float* w1, const float* b1, const float* w2, const float* b2,
                       int n, long long T, int dil, float rs, cudaStream_t stream) {
    constexpr size_t smem = ResH2<C>::smem;
    int sms = 0;
    if (int rc = set_max_smem_once<resblock_h2_kernel<C>>((int)smem)) return rc;
    if (int rc = sm_count(&sms)) return rc;
    const long long per_clip = (T + 15) / 16, total = per_clip * n;
    constexpr int WARPS = ResH2<C>::WARPS;
    const unsigned grid = (unsigned)std::min<long long>((total + WARPS - 1) / WARPS, sms);
    resblock_h2_kernel<C><<<grid, WARPS * 32, smem, stream>>>(x, out, w1, b1, w2, b2, T, dil, rs, per_clip, total);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------
// Tap-GEMM convolution with the same fp16 x 3 split, for the decoder-side convs BETWEEN the residual blocks (the k3 input
// conv of a DecoderConvBock, the two phases of its k4-s2 transposed convs, Decoder.out's wide cousins; encdec.py:28-46):
// out[t*os + oo, :] = res + scale * (sum_j x[t*is + off_j, :] . W_j + b), c_in, c_out in {32, 64}.
// One warp per 16 output positions like resblock_h2_kernel; weights (<= 4 taps) staged once per persistent CTA.
// ---------------------------------------------------------------------------------------
template <int CI, int CO>
struct ConvH2 {
    static constexpr int XA = CI + 8, XB = CO + 8, NT = CO / 8, WARPS = 16;
    static constexpr int w_halfs = 2 * 4 * CI * XB;
    static constexpr int warp_halfs = 2 * 16 * XA;         // one tap tile of a warp, hi and lo
    static constexpr size_t smem = (size_t)(w_halfs + WARPS * warp_halfs) * 2;
};

template <int CI, int CO>
__global__ void __launch_bounds__(512, 1) conv1d_h2_kernel(ConvP P, long long tiles_per_clip, long long total_tiles) {
    constexpr int XA = ConvH2<CI, CO>::XA, XB = ConvH2<CI, CO>::XB, NT = ConvH2<CI, CO>::NT, WARPS = ConvH2<CI, CO>::WARPS;
    extern __shared__ __align__(16) __half hsm[];
    const int ntap = P.n_taps;
    __half* wh = hsm;                           // [ntap * CI][XB]
    __half* wl = wh + 4 * CI * XB;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __half* xh = wl + 4 * CI * XB + warp * ConvH2<CI, CO>::warp_halfs;       // [16][XA]: the current tap's rows
    __half* xl = xh + 16 * XA;
    const int g = lane >> 2, t4 = lane & 3;
    for (int i = tid; i < ntap * CI * CO; i += WARPS * 32) {
        const int o = (i / CO) * XB + i % CO;
        split_f16(kWScale * __ldg(P.w + i), wh[o], wl[o]);
    }
    __syncthreads();
    constexpr int TX = CI / 4, PER = 16 * TX / 32, RJ = 32 / TX;
    const int lr = lane / TX, lc = lane % TX;
    const long long rows_out = P.t_out * P.out_stride;
    const int r = lane & 15, c8 = (lane >> 4) * 8;
    const long long stride = (long long)gridDim.x * WARPS;
    float4 v[PER];
    auto issue = [&](long long tile, int tap) {
        if (tile >= total_tiles) return;
        const long long nb = tile / tiles_per_clip, to = (tile - nb * tiles_per_clip) * 16 + lr;      // output row of j = 0
        const long long off = tap == 0 ? P.tap_off[0] : tap == 1 ? P.tap_off[1] : tap == 2 ? P.tap_off[2] : P.tap_off[3];
        const long long tb = to * P.in_stride + off;
        const float4* p = reinterpret_cast<const float4*>(P.in + ((size_t)nb * P.t_in + tb) * CI) + lc;
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            const long long tp = tb + (long long)j * RJ * P.in_stride;
            v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tp >= 0 && tp < P.t_in && to + j * RJ < P.t_out) v[j] = __ldg(p + (size_t)j * RJ * P.in_stride * TX);
        }
    };
    long long tile = (long long)blockIdx.x * WARPS + warp;
    issue(tile, 0);
#pragma unroll 1
    for (; tile < total_tiles; tile += stride) {
        const long long nb = tile / tiles_per_clip, t0 = (tile - nb * tiles_per_clip) * 16;
        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll 1
        for (int tap = 0; tap < ntap; ++tap) {
            __syncwarp();
#pragma unroll
            for (int j = 0; j < PER; ++j) {
                if (P.relu_in) { v[j].x = fmaxf(v[j].x, 0.f); v[j].y = fmaxf(v[j].y, 0.f); v[j].z = fmaxf(v[j].z, 0.f); v[j].w = fmaxf(v[j].w, 0.f); }
                uint2 h, l;
                split_f16x2(v[j].x, v[j].y, h.x, l.x);
                split_f16x2(v[j].z, v[j].w, h.y, l.y);
                *reinterpret_cast<uint2*>(xh + (lr + j * RJ) * XA + lc * 4) = h;
                *reinterpret_cast<uint2*>(xl + (lr + j * RJ) * XA + lc * 4) = l;
            }
            if (tap + 1 < ntap) issue(tile, tap + 1); else issue(tile + stride, 0);
            __syncwarp();
#pragma unroll
            for (int k16 = 0; k16 < CI / 16; ++k16) {
                uint32_t fh[4], fl[4];
                ldmatrix_x4(fh, xh + r * XA + k16 * 16 + c8);
                ldmatrix_x4(fl, xl + r * XA + k16 * 16 + c8);
                const __half* bh = wh + (tap * CI + k16 * 16 + r) * XB + c8;
                const __half* bl = wl + (tap * CI + k16 * 16 + r) * XB + c8;
#pragma unroll
                for (int np = 0; np < CO / 16; ++np) {
                    uint32_t qh[4], ql[4];
                    ldsm_x4_t(qh, bh + np * 16);
                    ldsm_x4_t(ql, bl + np * 16);
                    mma_16816(acc[2 * np], fl, qh[0], qh[1]);
                    mma_16816(acc[2 * np], fh, ql[0], ql[1]);
                    mma_16816(acc[2 * np], fh, qh[0], qh[1]);
                    mma_16816(acc[2 * np + 1], fl, qh[2], qh[3]);
                    mma_16816(acc[2 * np + 1], fh, ql[2], ql[3]);
                    mma_16816(acc[2 * np + 1], fh, qh[2], qh[3]);
                }
            }
        }
        float* out = P.out + (size_t)nb * rows_out * CO;
        const float* res = P.res ? P.res + (size_t)nb * rows_out * CO : nullptr;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const int col = nt * 8 + 2 * t4;
            float2 bv = make_float2(0.f, 0.f);
            if (P.bias) bv = __ldg(reinterpret_cast<const float2*>(P.bias + col));
#pragma unroll
            for (int hlf = 0; hlf < 2; ++hlf) {
                const long long t = t0 + g + 8 * hlf;
                if (t < P.t_out) {
                    const long long orow = t * P.out_stride + P.out_offset;
                    float2 o;
                    o.x = P.scale * fmaf(acc[nt][2 * hlf], kWInv, bv.x);
                    o.y = P.scale * fmaf(acc[nt][2 * hlf + 1], kWInv, bv.y);
                    if (res) {
                        const float2 rr = __ldg(reinterpret_cast<const float2*>(res + (size_t)orow * CO + col));
                        o.x += rr.x; o.y += rr.y;
                    }
                    *reinterpret_cast<float2*>(out + (size_t)orow * CO + col) = o;
                }
            }
        }
    }
}

template <int CI, int CO>
int launch_conv_h2(const ConvP& P, int n, cudaStream_t stream) {
    constexpr size_t smem = ConvH2<CI, CO>::smem;
    int sms = 0;
    if (int rc = set_max_smem_once<conv1d_h2_kernel<CI, CO>>((int)smem)) return rc;
    if (int rc = sm_count(&sms)) return rc;
    const long long per_clip = (P.t_out + 15) / 16, total = per_clip * n;
    constexpr int WARPS = ConvH2<CI, CO>::WARPS;
    const unsigned grid = (unsigned)std::min<long long>((total + WARPS - 1) / WARPS, sms);
    conv1d_h2_kernel<CI, CO><<<grid, WARPS * 32, smem, stream>>>(P, per_clip, total);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// c_out <= 4 (the decoder's final Conv1d(emb_width -> 1 audio channel, k3), encdec.py:109): one thread per output
// position, weights in shared memory.  The 64 x 64 tile kernel would spend 63/64 of its FMAs on padding here;
// this one is a stream over the input (HBM bound).  Same accumulation order as the tile kernel (tap, then channel).
__global__ void __launch_bounds__(256) conv1d_cl_narrow_kernel(ConvP P, int span, int min_off) {
    extern __shared__ __align__(16) float wsm[];         // [n_taps][c_in][c_out] | input rows [256 + span][c_in + 4]
    const int CI = P.c_in, CO = P.c_out, XS = CI + 4;
    const int nw = P.n_taps * CI * CO;
    float* xs = wsm + ((nw + 3) & ~3);
    for (int i = threadIdx.x; i < nw; i += 256) wsm[i] = P.w[i];
    const long long t0 = (long long)blockIdx.x * 256, t = t0 + threadIdx.x;
    const int nb = blockIdx.y;
    const float* in = P.in + (size_t)nb * P.t_in * CI;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int c4n = CI >> 2;
    // Input rows are loaded by the whole CTA with consecutive lanes on consecutive 16-byte chunks (one thread per output row
    // would touch 32 different rows per instruction), zero outside [0, t_in).  span >= 0: the taps of all 256 outputs lie in
    // one window of 256 + span rows (stride 1, small dilation: the decoder's output conv) - staged ONCE; else tap by tap.
    const int passes = span >= 0 ? 1 : P.n_taps;
    for (int pass = 0; pass < passes; ++pass) {
        __syncthreads();
        const long long off = span >= 0 ? min_off : (pass == 0 ? P.tap_off[0] : pass == 1 ? P.tap_off[1] : pass == 2 ? P.tap_off[2] : P.tap_off[3]);
        const int rows = span >= 0 ? 256 + span : 256;
        const int c4sh = (c4n & (c4n - 1)) == 0 ? 31 - __clz(c4n) : -1;      // c_in = 32 / 64: shifts, not a division per chunk
        if (!P.relu_in) {
            // cp.async (LDGSTS): every 16-byte chunk of the window is requested at once, nothing passes through registers -
            // the staging costs one memory round trip instead of a chain of load -> store batches; rows outside the clip are
            // zero-filled by the src-size operand
            for (int i = threadIdx.x; i < rows * c4n; i += 256) {
                const int r = c4sh >= 0 ? (i >> c4sh) : i / c4n, c4 = i - r * c4n;
                const long long tp = span >= 0 ? t0 + r + off : (t0 + r) * P.in_stride + off;
                const bool ok = tp >= 0 && tp < P.t_in;
                const float4* src = reinterpret_cast<const float4*>(in + (size_t)(ok ? tp : 0) * CI) + c4;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(xs + (size_t)r * XS + c4 * 4)),
                             "l"(src), "r"(ok ? 16 : 0) : "memory");
            }
            asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
        } else {
#pragma unroll 4
            for (int i = threadIdx.x; i < rows * c4n; i += 256) {
                const int r = c4sh >= 0 ? (i >> c4sh) : i / c4n, c4 = i - r * c4n;
                const long long tp = span >= 0 ? t0 + r + off : (t0 + r) * P.in_stride + off;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (tp >= 0 && tp < P.t_in) v = __ldg(reinterpret_cast<const float4*>(in + (size_t)tp * CI) + c4);
                v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
                *reinterpret_cast<float4*>(xs + (size_t)r * XS + c4 * 4) = v;
            }
        }
        __syncthreads();
        const int tap_lo = span >= 0 ? 0 : pass, tap_hi = span >= 0 ? P.n_taps : pass + 1;
        for (int tap = tap_lo; tap < tap_hi; ++tap) {
            const int toff = tap == 0 ? P.tap_off[0] : tap == 1 ? P.tap_off[1] : tap == 2 ? P.tap_off[2] : P.tap_off[3];
            const float* xr = xs + (size_t)(threadIdx.x + (span >= 0 ? toff - min_off : 0)) * XS;
            const float* wr = wsm + (size_t)tap * CI * CO;
            if (CO == 1) {      // the audio output conv: four weights per LDS.128 (was one broadcast LDS.32 per FMA); same order
#pragma unroll 4
                for (int c = 0; c < CI; c += 4) {
                    const float4 v = *reinterpret_cast<const float4*>(xr + c);
                    const float4 w4 = *reinterpret_cast<const float4*>(wr + c);
                    acc[0] = fmaf(v.x, w4.x, acc[0]); acc[0] = fmaf(v.y, w4.y, acc[0]);
                    acc[0] = fmaf(v.z, w4.z, acc[0]); acc[0] = fmaf(v.w, w4.w, acc[0]);
                }
                continue;
            }
            for (int c = 0; c < CI; c += 4) {            // same accumulation order as the tile kernel: tap, then channel
                const float4 v = *reinterpret_cast<const float4*>(xr + c);
                const float xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (j < CO) acc[j] = fmaf(xv[e], wr[(c + e) * CO + j], acc[j]);
            }
        }
    }
    if (t >= P.t_out) return;
    const long long rows_out = P.t_out * P.out_stride;
    const long long orow = t * P.out_stride + P.out_offset;
    float* out = P.out + ((size_t)nb * rows_out + orow) * CO;
    const float* res = P.res ? P.res + ((size_t)nb * rows_out + orow) * CO : nullptr;
    for (int j = 0; j < CO; ++j) {
        float v = P.scale * (acc[j] + (P.bias ? P.bias[j] : 0.f));
        if (res) v += res[j];
        out[j] = v;
    }
}

__global__ void pack_conv_weight_kernel(const float* __restrict__ w, float* __restrict__ packed, int c_out, int c_in,
                                        int k, int transposed) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int total = c_out * c_in * k;
    if (i >= total) return;
    const int co = i % c_out, ci = (i / c_out) % c_in, kk = i / (c_out * c_in);
    const size_t src = transposed ? ((size_t)ci * c_out + co) * k + kk : ((size_t)co * c_in + ci) * k + kk;
    packed[i] = w[src];
}

__global__ void layernorm_f32_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ b,
                                     float* __restrict__ y, long long rows, int width, float eps) {
    __shared__ float sh[8];
    const long long r = blockIdx.x;
    const float* xr = x + r * width;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float s = 0.f;
    for (int i = tid; i < width; i += 256) s += xr[i];
    s = warp_sum(s);
    if (lane == 0) sh[warp] = s;
    __syncthreads();
    float mean = 0.f;
    for (int w = 0; w < 8; ++w) mean += sh[w];
    mean /= (float)width;
    __syncthreads();
    float ss = 0.f;
    for (int i = tid; i < width; i += 256) { float d = xr[i] - mean; ss += d * d; }
    ss = warp_sum(ss);
    if (lane == 0) sh[warp] = ss;
    __syncthreads();
    float var = 0.f;
    for (int w = 0; w < 8; ++w) var += sh[w];
    const float rstd = 1.0f / sqrtf(var / (float)width + eps);
    for (int i = tid; i < width; i += 256) y[r * width + i] = (xr[i] - mean) * rstd * g[i] + b[i];
}

__global__ void embedding_f32_kernel(const long long* __restrict__ idx, const float* __restrict__ table,
                                     const float* __restrict__ add, float* __restrict__ out, long long n, int rows,
                                     int width) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * width) return;
    const long long r = i / width;
    const int d = (int)(i % width);
    long long j = idx[r];
    j = j < 0 ? 0 : (j >= rows ? rows - 1 : j);
    float v = table[j * width + d];
    if (add) v += add[i];
    out[i] = v;
}

}  // namespace

extern "C" int jk_vq_argmin(const float* x, const float* codebook, int64_t* idx, float* min_dist, int64_t n, int k_bins,
                            int width, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(x && codebook && idx, "null argument");
    JK_REQUIRE(n >= 0 && k_bins >= 1 && width >= 1, "bad sizes");
    if (n == 0) return 0;
    if (width == 64) {
        vq_argmin_kernel<64><<<(unsigned)((n + 63) / 64), 256, 0, stream>>>(x, codebook, (long long*)idx, min_dist, n, k_bins);
    } else {
        vq_argmin_generic_kernel<<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(x, codebook, (long long*)idx, min_dist, n, k_bins, width);
    }
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_vq_gather(const int64_t* idx, const float* codebook, float* out, int64_t n, int k_bins, int width,
                            jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(idx && codebook && out, "null argument");
    JK_REQUIRE(width % 4 == 0, "width must be a multiple of 4");
    if (n == 0) return 0;
    const long long total = n * (width / 4);
    vq_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>((const long long*)idx, codebook, out, n, k_bins, width / 4);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

namespace jk {
int conv_t5(const float* in, long long t_in, int c_in, float* out, long long t_out, int c_out, const float* w, const float* bias,
            const float* res, int n_taps, const int* tap_off, int out_stride, int out_offset, int relu_in, float scale, int n,
            cudaStream_t stream);                                                 // vqvae_t5.cu
int resblock_t5(const float* x, float* out, const float* w1, const float* b1, const float* w2, const float* b2, int n,
                long long T, int C, int dil, float rs, cudaStream_t stream);      // vqvae_t5.cu
int conv_wide_t5(const float* in, long long t_in, int c_in, float* out, long long t_out, int c_out, const void* w_split,
                 const float* bias, const float* res, int n_taps, const int* tap_off, int out_stride, int out_offset,
                 int relu_in, float scale, int n, cudaStream_t stream);       // vqvae_t5.cu
int pack_conv_weight_split(const float* packed, void* split, int k, int c_in, int c_out, cudaStream_t stream);   // vqvae_t5.cu
}

extern "C" int jk_conv1d_cl(const jk_conv_args* a, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(a && a->in && a->out && a->w, "null argument");
    JK_REQUIRE(a->n_taps >= 1 && a->n_taps <= 4, "n_taps must be 1..4");
    JK_REQUIRE(a->n >= 1 && a->n <= 65535, "batch out of range");
    JK_REQUIRE(a->in_stride >= 1 && a->out_stride >= 1, "bad strides");
    if (a->t_out == 0) return 0;
    ConvP P;
    P.in = a->in; P.t_in = a->t_in; P.c_in = a->c_in; P.out = a->out; P.t_out = a->t_out; P.c_out = a->c_out;
    P.w = a->w; P.bias = a->bias; P.res = a->res; P.n_taps = a->n_taps;
    for (int i = 0; i < 4; ++i) P.tap_off[i] = a->tap_off[i];
    P.in_stride = a->in_stride; P.out_stride = a->out_stride; P.out_offset = a->out_offset; P.relu_in = a->relu_in;
    P.scale = a->scale;
    if (a->c_out <= 4 && a->c_in % 4 == 0 && a->c_in <= 128 && ((uintptr_t)a->in & 15) == 0 &&
        (size_t)a->n_taps * a->c_in * a->c_out * 4 <= 32768) {
        dim3 g((unsigned)((a->t_out + 255) / 256), (unsigned)a->n);
        int lo = a->tap_off[0], hi = a->tap_off[0];
        for (int i = 1; i < a->n_taps; ++i) { lo = std::min(lo, (int)a->tap_off[i]); hi = std::max(hi, (int)a->tap_off[i]); }
        const int span = (a->in_stride == 1 && hi - lo <= 16) ? hi - lo : -1;        // one staging window covers every tap
        const size_t nsm = (((size_t)a->n_taps * a->c_in * a->c_out + 3) & ~(size_t)3) * 4 +
                           (size_t)(256 + std::max(span, 0)) * (a->c_in + 4) * 4;
        if (int rc = set_max_smem_once<conv1d_cl_narrow_kernel>(200 * 1024)) return rc;
        conv1d_cl_narrow_kernel<<<g, 256, nsm, stream>>>(P, span, lo);
        JK_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    if (a->tensor_cores && (a->c_in == 32 || a->c_in == 64) && (a->c_out == 32 || a->c_out == 64) &&
        (((uintptr_t)a->in | (uintptr_t)a->out | (uintptr_t)a->bias | (uintptr_t)a->res) & 15) == 0) {
        // wgmma + TMA tap-GEMM (vqvae_t5.cu) for stride-1 inputs of >= 128 positions, the mma.sync kernel for the rest
        if (a->in_stride == 1 && a->n_taps <= 3 && a->t_in >= 128 && a->t_out >= 1)
            return jk::conv_t5(a->in, a->t_in, a->c_in, a->out, a->t_out, a->c_out, a->w, a->bias, a->res, a->n_taps, a->tap_off,
                               a->out_stride, a->out_offset, a->relu_in, a->scale, a->n, stream);
        if (a->c_in == 64 && a->c_out == 64) return launch_conv_h2<64, 64>(P, a->n, stream);
        if (a->c_in == 64 && a->c_out == 32) return launch_conv_h2<64, 32>(P, a->n, stream);
        if (a->c_in == 32 && a->c_out == 64) return launch_conv_h2<32, 64>(P, a->n, stream);
        return launch_conv_h2<32, 32>(P, a->n, stream);
    }
    if ((a->c_out == 64 || a->c_out == 32) && a->c_in % 4 == 0 && a->c_in >= 4 && a->c_in <= 64 &&
        (((uintptr_t)a->in | (uintptr_t)a->out | (uintptr_t)a->w | (uintptr_t)a->bias | (uintptr_t)a->res) & 15) == 0) {
        bool took = false;
        const int rc = a->c_out == 64 ? launch_conv_tile<64>(P, a->n, stream, &took) : launch_conv_tile<32>(P, a->n, stream, &took);
        if (rc) return rc;
        if (took) return 0;
    }
    dim3 grid((unsigned)((a->t_out + 63) / 64), (unsigned)((a->c_out + 63) / 64), (unsigned)a->n);
    conv1d_cl_kernel<<<grid, 256, 0, stream>>>(P);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_resblock_cl(const float* x, float* out, float* tmp, const float* w1, const float* b1, const float* w2,
                              const float* b2, int n, int64_t T, int C, int Cs, int dilation, float res_scale,
                              jk_stream_t stream) {
    JK_REQUIRE(x && out && w1 && w2, "null argument");
    // the fused kernel reads x, w1, w2, b1, b2 and writes out as float4: other pointers take the two launches below, whose
    // dispatch checks alignment before every vector access
    const bool vec4 = (((uintptr_t)x | (uintptr_t)out | (uintptr_t)w1 | (uintptr_t)w2 | (uintptr_t)b1 | (uintptr_t)b2) & 15) == 0;
    if (C == Cs && b1 && b2 && x != out && T > 0 && vec4) {   // the VQ-VAE's own shapes: one fused launch
        if (C == 64) return launch_resblock_fused<64>(x, out, w1, b1, w2, b2, n, T, dilation, res_scale, (cudaStream_t)stream);
        if (C == 32) return launch_resblock_fused<32>(x, out, w1, b1, w2, b2, n, T, dilation, res_scale, (cudaStream_t)stream);
    }
    JK_REQUIRE(tmp, "jk_resblock_cl: tmp ([n, T, Cs] floats) is required unless C == Cs in {32, 64} and x, out, w1, w2, b1, b2 "
                    "are 16-byte aligned (the fused kernel)");
    jk_conv_args a;
    a.tensor_cores = 0;
    a.in = x; a.t_in = T; a.c_in = C; a.out = tmp; a.t_out = T; a.c_out = Cs; a.w = w1; a.bias = b1; a.res = nullptr;
    a.n_taps = 3; a.tap_off[0] = -dilation; a.tap_off[1] = 0; a.tap_off[2] = dilation; a.tap_off[3] = 0;
    a.in_stride = 1; a.out_stride = 1; a.out_offset = 0; a.relu_in = 1; a.scale = 1.0f; a.n = n;
    int rc = jk_conv1d_cl(&a, stream);
    if (rc) return rc;
    a.in = tmp; a.c_in = Cs; a.out = out; a.c_out = C; a.w = w2; a.bias = b2; a.res = x; a.n_taps = 1; a.tap_off[0] = 0;
    a.scale = res_scale;
    return jk_conv1d_cl(&a, stream);
}


extern "C" int jk_resblock_tc(const float* x, float* out, const float* w1, const float* b1, const float* w2, const float* b2,
                              int n, int64_t T, int C, int dilation, float res_scale, jk_stream_t stream) {
    JK_REQUIRE(x && out && w1 && w2 && b1 && b2, "null argument");
    JK_REQUIRE(x != out && T > 0 && n > 0, "x and out must differ, T and n must be positive");
    // both kernels read x and write out in 16-byte (t5) or 8- and 16-byte (h2) vectors, and the h2 kernel reads b1 / b2 as float2
    JK_REQUIRE((((uintptr_t)x | (uintptr_t)out) & 15) == 0 && (((uintptr_t)b1 | (uintptr_t)b2) & 7) == 0,
               "jk_resblock_tc: x and out must be 16-byte aligned, b1 and b2 8-byte aligned");
    // wgmma + TMA version (vqvae_t5.cu): whole 128-position MMA tiles
    if ((C == 64 || C == 32) && T >= 128)
        return jk::resblock_t5(x, out, w1, b1, w2, b2, n, T, C, dilation, res_scale, (cudaStream_t)stream);
    if (C == 64) return launch_resblock_h2<64>(x, out, w1, b1, w2, b2, n, T, dilation, res_scale, (cudaStream_t)stream);
    if (C == 32) return launch_resblock_h2<32>(x, out, w1, b1, w2, b2, n, T, dilation, res_scale, (cudaStream_t)stream);
    JK_REQUIRE(false, "jk_resblock_tc: C must be 32 or 64 (got %d)", C);
    return 0;
}

extern "C" int jk_pack_conv_weight(const float* w, float* packed, int c_out, int c_in, int k, int transposed,
                                   jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(w && packed, "null argument");
    const int total = c_out * c_in * k;
    pack_conv_weight_kernel<<<(total + 255) / 256, 256, 0, stream>>>(w, packed, c_out, c_in, k, transposed);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_conv_weight_split_bytes(int k, int c_in, int c_out, size_t* bytes) {
    JK_REQUIRE(bytes, "null argument");
    JK_REQUIRE(k >= 1 && c_in >= 1 && c_out >= 1, "k, c_in and c_out must be positive");
    *bytes = (size_t)2 * k * c_in * c_out * 2;
    return 0;
}

extern "C" int jk_pack_conv_weight_split(const float* packed, void* split, int k, int c_in, int c_out, jk_stream_t stream) {
    JK_REQUIRE(packed && split, "null argument");
    JK_REQUIRE(k >= 1 && c_in >= 1 && c_out >= 1, "k, c_in and c_out must be positive");
    return jk::pack_conv_weight_split(packed, split, k, c_in, c_out, (cudaStream_t)stream);
}

extern "C" int jk_conv1d_tc_wide(const jk_conv_args* a, const void* w_split, jk_stream_t stream) {
    JK_REQUIRE(a && a->in && a->out && w_split, "null argument");
    JK_REQUIRE(a->c_in % 64 == 0 && a->c_out % 64 == 0 && a->c_in > 0 && a->c_out > 0 && (a->c_in > 64 || a->c_out > 64),
               "jk_conv1d_tc_wide: c_in and c_out must be multiples of 64 and one of them above 64 (got %d -> %d)", a->c_in, a->c_out);
    JK_REQUIRE(a->in_stride == 1, "jk_conv1d_tc_wide: the input stride must be 1 (got %d)", a->in_stride);
    JK_REQUIRE(a->n_taps >= 1 && a->n_taps <= 3, "jk_conv1d_tc_wide: n_taps must be 1..3 (got %d)", a->n_taps);
    JK_REQUIRE(a->t_in >= 128, "jk_conv1d_tc_wide: t_in must be at least 128 positions (got %lld)", (long long)a->t_in);
    JK_REQUIRE(a->n >= 1 && a->n <= 65535, "jk_conv1d_tc_wide: batch out of range");
    JK_REQUIRE(a->out_stride >= 1 && a->out_offset >= 0 && a->out_offset < a->out_stride, "jk_conv1d_tc_wide: bad output stride / offset");
    JK_REQUIRE((((uintptr_t)a->in | (uintptr_t)a->out | (uintptr_t)a->bias | (uintptr_t)a->res | (uintptr_t)w_split) & 15) == 0,
               "jk_conv1d_tc_wide: in, out, bias, res and w_split must be 16-byte aligned");
    if (a->t_out == 0) return 0;
    return jk::conv_wide_t5(a->in, a->t_in, a->c_in, a->out, a->t_out, a->c_out, w_split, a->bias, a->res, a->n_taps, a->tap_off,
                            a->out_stride, a->out_offset, a->relu_in, a->scale, a->n, (cudaStream_t)stream);
}

extern "C" int jk_layernorm_f32(const float* x, const float* g, const float* b, float* y, int64_t rows, int width,
                                float eps, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(x && g && b && y, "null argument");
    if (rows == 0) return 0;
    JK_REQUIRE(rows < (1ll << 31), "too many rows");
    layernorm_f32_kernel<<<(unsigned)rows, 256, 0, stream>>>(x, g, b, y, rows, width, eps);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_embedding_f32(const int64_t* idx, const float* table, const float* add, float* out, int64_t n, int rows,
                                int width, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(idx && table && out, "null argument");
    if (n == 0) return 0;
    const long long total = n * width;
    embedding_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>((const long long*)idx, table, add, out, n, rows, width);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}
