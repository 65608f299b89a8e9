// Gradients of the fp32 transformer path (csrc/f32_path.cu forward mode) for fine-tuning a prior's decoder.
//
// jk_f32_backward walks the layers depth-1 .. 0.  Only each layer's input is kept from the forward; the layer's
// intermediates are recomputed from it (LN0, qkv, attention, x1, LN1, the fc pre-activation and g) with the same
// arithmetic as jk_f32_forward, then differentiated:
//   h = x1 + gelu(LN1(x1) . fc) . proj2,  x1 = x + attn(LN0(x) . c_attn) . c_proj        (transformer.py:82-83)
// Every kernel here is deterministic: each output element is written by one thread with a fixed summation order
// (warp shuffles, fixed-order shared-memory reductions, row-serial loops).  No atomics touch a floating-point sum, so
// two identical calls give bit-identical gradients.
//
// Attention backward is two passes over the layer's pattern (the key sets of f32_path.cu's f32_nkeys / f32_key):
//   query pass - one CTA per (query, head, item): recomputes the row's scores, writes its log-sum-exp, D = dO . O and
//                dQ = scale^2 . sum_j dS_j k_j;
//   key pass   - one CTA per (key, head, item): walks the queries that attend the key (the inverse key set), recomputes
//                p = exp(s - lse) and dS = p (dO . v - D) from the saved row statistics, and sums dV = sum p dO and
//                dK = scale^2 sum dS q in registers.
// The input gradient of a Conv1D, dX = dY . W^T, is the forward's sgemm in its [N, K] weight mode (jk_f32_linear).
#include <assert.h>
#include <math.h>

#include "common.cuh"
#include "../../include/jkb200.h"

namespace {

// ---- key sets of the six patterns over a whole window (p0 = 0, P = n_ctx) -------------------------------------------
struct AttnG {
    const float* q;  int q_stride;                    // query rows [b * P + i]
    const float* k;  const float* v;  int kv_stride;  // key rows [b * Lk + r]
    const float* o;                                   // [M, S] attention output (recomputed forward)
    const float* dout;                                // [M, S] dL/dO
    float* o_w;                                       // forward recompute writes O here
    float* lse;  float* dd;                           // [n, H, P] row log-sum-exp and D = dO . O
    float* dq;   int dq_stride;
    float* dk;   float* dv;  int dkv_stride;          // key-row gradients [b * Lk + r]
    int P, S, H, dh, bc, attn_func, prime, Lk;
    float scale2;
};

// keys of query p: the same sets as f32_path.cu (f32_nkeys / f32_key) with p0 = 0 and caches of the whole window
__device__ __forceinline__ int g_nkeys(const AttnG& A, int p) {
    switch (A.attn_func) {
        case 0: return p + 1;
        case 1: return p % A.bc + 1;
        case 2: return p / A.bc + 1;
        case 3: return p >= A.bc ? A.bc : 0;
        case 6: return A.Lk;
        case 7: return p < A.prime ? p + 1 : A.prime;
    }
    return 0;
}
__device__ __forceinline__ int g_key(const AttnG& A, int p, int j) {
    switch (A.attn_func) {
        case 1: return p - p % A.bc + j;
        case 2: return p % A.bc + j * A.bc;
        case 3: return (p / A.bc - 1) * A.bc + j;
    }
    return j;
}
// the inverse sets: queries that attend key row r
//   dense / prime: p >= r (prime: only rows r < prime are cached, kv_store_kernel's limit); block: p >= r in r's block;
//   transpose: same offset in r's block or a later one; previous-block: every query of the next block; enc-dec: all.
__device__ __forceinline__ int g_nqueries(const AttnG& A, int r) {
    switch (A.attn_func) {
        case 0: return A.P - r;
        case 1: return A.bc - r % A.bc;
        case 2: return (A.P - 1 - r) / A.bc + 1;
        case 3: return (r / A.bc + 1) * A.bc < A.P ? A.bc : 0;
        case 6: return A.P;
        case 7: return r < A.prime ? A.P - r : 0;
    }
    return 0;
}
__device__ __forceinline__ int g_query(const AttnG& A, int r, int j) {
    switch (A.attn_func) {
        case 2: return r + j * A.bc;
        case 3: return (r / A.bc + 1) * A.bc + j;
        case 6: return j;
    }
    return r + j;   // 0, 1, 7
}

// ---- attention forward, recomputed: O of every query (the arithmetic of attn_f32_kernel) -----------------------------
__global__ void __launch_bounds__(128) attn_fwd_kernel(AttnG A) {
    extern __shared__ float fsm[];
    float* qs = fsm;
    float* sc = fsm + A.dh;
    __shared__ float red[4];
    const int i = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dh = A.dh;
    const size_t row = (size_t)b * A.P + i;
    float* out = A.o_w + row * A.S + h * dh;
    const int nk = g_nkeys(A, i);
    if (nk == 0) {
        for (int d = tid; d < dh; d += 128) out[d] = 0.f;
        return;
    }
    for (int d = tid; d < dh; d += 128) qs[d] = A.q[row * A.q_stride + h * dh + d];
    __syncthreads();
    const float* kb = A.k + (size_t)b * A.Lk * A.kv_stride + h * dh;
    const float* vb = A.v + (size_t)b * A.Lk * A.kv_stride + h * dh;
    for (int j = warp; j < nk; j += 4) {
        const float* k = kb + (size_t)g_key(A, i, j) * A.kv_stride;
        float dot = 0.f;
        for (int d = lane; d < dh; d += 32) dot = fmaf(qs[d], k[d], dot);
        dot = jk::warp_sum(dot);
        if (lane == 0) sc[j] = dot * A.scale2;
    }
    __syncthreads();
    float mx = -INFINITY;
    for (int j = tid; j < nk; j += 128) mx = fmaxf(mx, sc[j]);
    mx = jk::warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    __syncthreads();
    float l = 0.f;
    for (int j = tid; j < nk; j += 128) {
        const float e = expf(sc[j] - mx);
        l += e;
        sc[j] = e;
    }
    l = jk::warp_sum(l);
    if (lane == 0) red[warp] = l;
    __syncthreads();
    const float inv = 1.f / (red[0] + red[1] + red[2] + red[3]);
    for (int d = tid; d < dh; d += 128) {
        float o = 0.f;
        for (int j = 0; j < nk; ++j) o = fmaf(sc[j] * inv, vb[(size_t)g_key(A, i, j) * A.kv_stride + d], o);
        out[d] = o;
    }
}

// ---- attention backward, query pass ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) attn_bwd_query_kernel(AttnG A) {
    extern __shared__ float fsm[];
    float* qs = fsm;                 // [dh]
    float* dos = fsm + A.dh;         // [dh]
    float* sc = fsm + 2 * A.dh;      // [nk]: scores, then probabilities, then dS
    __shared__ float red[4];
    const int i = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dh = A.dh;
    const size_t row = (size_t)b * A.P + i;
    const size_t stat = ((size_t)b * A.H + h) * A.P + i;
    float* dq = A.dq + row * A.dq_stride + h * dh;
    const int nk = g_nkeys(A, i);
    if (nk == 0) {      // a previous-block query of the first block: no keys, output 0, no gradient
        for (int d = tid; d < dh; d += 128) dq[d] = 0.f;
        if (tid == 0) A.lse[stat] = A.dd[stat] = 0.f;
        return;
    }
    float dsum = 0.f;
    for (int d = tid; d < dh; d += 128) {
        qs[d] = A.q[row * A.q_stride + h * dh + d];
        const float g = A.dout[row * A.S + h * dh + d];
        dos[d] = g;
        dsum = fmaf(g, A.o[row * A.S + h * dh + d], dsum);
    }
    dsum = jk::warp_sum(dsum);
    if (lane == 0) red[warp] = dsum;
    __syncthreads();
    const float D = (red[0] + red[1]) + (red[2] + red[3]);
    __syncthreads();
    const float* kb = A.k + (size_t)b * A.Lk * A.kv_stride + h * dh;
    const float* vb = A.v + (size_t)b * A.Lk * A.kv_stride + h * dh;
    for (int j = warp; j < nk; j += 4) {
        const float* k = kb + (size_t)g_key(A, i, j) * A.kv_stride;
        float dot = 0.f;
        for (int d = lane; d < dh; d += 32) dot = fmaf(qs[d], k[d], dot);
        dot = jk::warp_sum(dot);
        if (lane == 0) sc[j] = dot * A.scale2;
    }
    __syncthreads();
    float mx = -INFINITY;
    for (int j = tid; j < nk; j += 128) mx = fmaxf(mx, sc[j]);
    mx = jk::warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    __syncthreads();
    float l = 0.f;
    for (int j = tid; j < nk; j += 128) {
        const float e = expf(sc[j] - mx);
        l += e;
        sc[j] = e;
    }
    l = jk::warp_sum(l);
    if (lane == 0) red[warp] = l;
    __syncthreads();
    const float lsum = red[0] + red[1] + red[2] + red[3];
    const float inv = 1.f / lsum;
    for (int j = warp; j < nk; j += 4) {
        const float* v = vb + (size_t)g_key(A, i, j) * A.kv_stride;
        float dp = 0.f;
        for (int d = lane; d < dh; d += 32) dp = fmaf(dos[d], v[d], dp);
        dp = jk::warp_sum(dp);
        if (lane == 0) sc[j] = sc[j] * inv * (dp - D);
    }
    __syncthreads();
    for (int d = tid; d < dh; d += 128) {
        float acc = 0.f;
        for (int j = 0; j < nk; ++j) acc = fmaf(sc[j], kb[(size_t)g_key(A, i, j) * A.kv_stride + d], acc);
        dq[d] = acc * A.scale2;
    }
    if (tid == 0) {
        A.lse[stat] = mx + logf(lsum);
        A.dd[stat] = D;
    }
}

#ifdef JK_F32_GRAD_DEBUG
// debug builds: the key pass checks every query it visits against the query pass's key set
__device__ bool g_attends(const AttnG& A, int p, int r) {
    const int nk = g_nkeys(A, p);
    for (int j = 0; j < nk; ++j)
        if (g_key(A, p, j) == r) return true;
    return false;
}
#endif

// ---- attention backward, key pass ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) attn_bwd_key_kernel(AttnG A) {
    extern __shared__ float fsm[];
    float* ks = fsm;                 // [dh]
    float* vs = fsm + A.dh;          // [dh]
    float* pj = fsm + 2 * A.dh;      // [nq]
    float* dsj = pj + A.P;           // [nq]
    const int r = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dh = A.dh;
    const size_t krow = (size_t)b * A.Lk + r;
    float* dk = A.dk + krow * A.dkv_stride + h * dh;
    float* dv = A.dv + krow * A.dkv_stride + h * dh;
    const int nq = g_nqueries(A, r);
    for (int d = tid; d < dh; d += 128) {
        ks[d] = A.k[krow * A.kv_stride + h * dh + d];
        vs[d] = A.v[krow * A.kv_stride + h * dh + d];
    }
    __syncthreads();
    for (int j = warp; j < nq; j += 4) {
        const int p = g_query(A, r, j);
#ifdef JK_F32_GRAD_DEBUG
        assert(p >= 0 && p < A.P && g_attends(A, p, r));
#endif
        const size_t qrow = (size_t)b * A.P + p;
        const float* q = A.q + qrow * A.q_stride + h * dh;
        const float* go = A.dout + qrow * A.S + h * dh;
        float s = 0.f, dp = 0.f;
        for (int d = lane; d < dh; d += 32) {
            s = fmaf(q[d], ks[d], s);
            dp = fmaf(go[d], vs[d], dp);
        }
        s = jk::warp_sum(s);
        dp = jk::warp_sum(dp);
        if (lane == 0) {
            const size_t stat = ((size_t)b * A.H + h) * A.P + p;
            const float pr = expf(s * A.scale2 - A.lse[stat]);
            pj[j] = pr;
            dsj[j] = pr * (dp - A.dd[stat]);
        }
    }
    __syncthreads();
    for (int d = tid; d < dh; d += 128) {
        float gv = 0.f, gk = 0.f;
        for (int j = 0; j < nq; ++j) {
            const size_t qrow = (size_t)b * A.P + g_query(A, r, j);
            gv = fmaf(pj[j], A.dout[qrow * A.S + h * dh + d], gv);
            gk = fmaf(dsj[j], A.q[qrow * A.q_stride + h * dh + d], gk);
        }
        dv[d] = gv;
        dk[d] = gk * A.scale2;
    }
}

// ---- dW[K, N] (+)= X^T . dY over M rows ----------------------------------------------------------------------------------
// 64 x 64 tile of dW per CTA, the whole M reduction in one CTA (rows in order, 16 at a time): no split, no atomics.
__global__ void __launch_bounds__(256) wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* dw,
                                                    int M, int K, int N, int accumulate) {
    __shared__ float xs[16][64 + 4];     // [m][k]
    __shared__ float gs[16][64 + 4];     // [m][n]
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int k0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int m0 = 0; m0 < M; m0 += 16) {
        for (int i = tid; i < 16 * 64; i += 256) {
            const int m = i >> 6, c = i & 63;
            const bool in = m0 + m < M;
            xs[m][c] = (in && k0 + c < K) ? x[(size_t)(m0 + m) * K + k0 + c] : 0.f;
            gs[m][c] = (in && n0 + c < N) ? dy[(size_t)(m0 + m) * N + n0 + c] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int m = 0; m < 16; ++m) {
            float a[4], g[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = xs[m][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) g[j] = gs[m][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], g[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int k = k0 + ty * 4 + i;
        if (k >= K) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float* o = dw + (size_t)k * N + n;
            *o = accumulate ? *o + acc[i][j] : acc[i][j];
        }
    }
}

// ---- column sums over rows: db[N] (+)= sum_m dY[m, :]; with x / mu / rstd also LayerNorm's dgamma -------------------
// One CTA per 32 columns: eight row groups each sum rows g, g + 8, ... in order, then one thread adds the eight partial
// sums in order (the two stages of a fixed-order reduction).
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                     const float* __restrict__ stats, float* db, float* dg, int M, int N,
                                                     int accumulate) {
    __shared__ float pb[8][33], pg[8][33];
    const int c = blockIdx.x * 32 + (threadIdx.x & 31), grp = threadIdx.x >> 5;
    float sb = 0.f, sg = 0.f;
    if (c < N) {
        for (int m = grp; m < M; m += 8) {
            const float g = dy[(size_t)m * N + c];
            sb += g;
            if (x) sg = fmaf(g, (x[(size_t)m * N + c] - stats[2 * m]) * stats[2 * m + 1], sg);
        }
    }
    pb[grp][threadIdx.x & 31] = sb;
    pg[grp][threadIdx.x & 31] = sg;
    __syncthreads();
    if (grp == 0 && c < N) {
        float tb = 0.f, tg = 0.f;
        for (int i = 0; i < 8; ++i) {
            tb += pb[i][threadIdx.x];
            tg += pg[i][threadIdx.x];
        }
        if (db) db[c] = accumulate ? db[c] + tb : tb;
        if (dg) dg[c] = accumulate ? dg[c] + tg : tg;
    }
}

// ---- LayerNorm backward, per row: dx (+)= rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat)), dxhat = dy . gamma ----
// Row statistics as layernorm_f32_kernel computes them (biased variance, eps inside the root), saved for dgamma.
__global__ void __launch_bounds__(256) ln_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                     const float* __restrict__ dy, float* dx, float* stats, int W,
                                                     float eps, int accumulate) {
    __shared__ float sh[8], sh2[8];
    const size_t r = blockIdx.x;
    const float* xr = x + r * W;
    const float* gr = dy + r * W;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float s = 0.f;
    for (int i = tid; i < W; i += 256) s += xr[i];
    s = jk::warp_sum(s);
    if (lane == 0) sh[warp] = s;
    __syncthreads();
    float mean = 0.f;
    for (int w = 0; w < 8; ++w) mean += sh[w];
    mean /= (float)W;
    __syncthreads();
    float ss = 0.f;
    for (int i = tid; i < W; i += 256) { const float d = xr[i] - mean; ss += d * d; }
    ss = jk::warp_sum(ss);
    if (lane == 0) sh[warp] = ss;
    __syncthreads();
    float var = 0.f;
    for (int w = 0; w < 8; ++w) var += sh[w];
    const float rstd = 1.0f / sqrtf(var / (float)W + eps);
    __syncthreads();
    float a = 0.f, bsum = 0.f;        // sum dxhat, sum dxhat * xhat
    for (int i = tid; i < W; i += 256) {
        const float dxh = gr[i] * gamma[i];
        a += dxh;
        bsum = fmaf(dxh, (xr[i] - mean) * rstd, bsum);
    }
    a = jk::warp_sum(a);
    bsum = jk::warp_sum(bsum);
    if (lane == 0) { sh[warp] = a; sh2[warp] = bsum; }
    __syncthreads();
    float ma = 0.f, mb = 0.f;
    for (int w = 0; w < 8; ++w) { ma += sh[w]; mb += sh2[w]; }
    ma /= (float)W;
    mb /= (float)W;
    for (int i = tid; i < W; i += 256) {
        const float xh = (xr[i] - mean) * rstd;
        const float v = rstd * (gr[i] * gamma[i] - ma - xh * mb);
        dx[r * W + i] = accumulate ? dx[r * W + i] + v : v;
    }
    if (tid == 0) { stats[2 * r] = mean; stats[2 * r + 1] = rstd; }
}

// ---- elementwise ---------------------------------------------------------------------------------------------------
__global__ void add_kernel(float* y, const float* __restrict__ a, size_t cnt) {       // y += a
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < cnt) y[i] += a[i];
}
__global__ void gelu_kernel(const float* __restrict__ a, float* g, size_t cnt) {       // f32_path's F32_EPI_GELU
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < cnt) { const float v = a[i]; g[i] = v * (1.0f / (1.0f + expf(-1.702f * v))); }
}
// dG -> dA in place: quick_gelu'(a) = s (1 + 1.702 a (1 - s)), s = sigmoid(1.702 a)
__global__ void gelu_bwd_kernel(const float* __restrict__ a, float* dg, size_t cnt) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    const float v = a[i];
    const float s = 1.0f / (1.0f + expf(-1.702f * v));
    dg[i] *= s * (1.0f + 1.702f * v * (1.0f - s));
}
// the c_enc_kv output [rows, 2S] <-> separate K / V gradients [rows, S]
__global__ void merge_kv_kernel(const float* __restrict__ dk, const float* __restrict__ dv, float* dkv, size_t rows, int S) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * S) return;
    const size_t r = i / S;
    const int s = (int)(i % S);
    dkv[r * 2 * S + s] = dk[i];
    dkv[r * 2 * S + S + s] = dv[i];
}

// ---- embedding backward --------------------------------------------------------------------------------------------
// The (token, row) pairs of positions t >= 1 get unique keys token * M + row; each pair's rank among all keys is its
// slot in the sorted order, so the sort is deterministic without any ordering among equal tokens to settle.
__global__ void rank_sort_kernel(const long long* __restrict__ tokens, long long tok_stride, int n, int P,
                                 int* sorted_rows, int* sorted_tok) {
    const int cnt = n * (P - 1);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    const int M = n * P;
    auto key = [&](int j) -> long long {
        const int b = j / (P - 1), t = j % (P - 1) + 1;
        return tokens[(size_t)b * tok_stride + t - 1] * (long long)M + (long long)b * P + t;
    };
    const long long ki = key(i);
    int rank = 0;
    for (int j = 0; j < cnt; ++j) rank += key(j) < ki;
    sorted_rows[rank] = (int)(ki % M);
    sorted_tok[rank] = (int)(ki / M);
}
// d x_emb[id, c] (+)= sum over the id's rows, in row order.  One thread per (id, column).
__global__ void emb_reduce_kernel(const float* __restrict__ dh, const int* __restrict__ sorted_rows,
                                  const int* __restrict__ sorted_tok, int cnt, float* dtab, int bins, int W, int accumulate) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, id = blockIdx.y;
    if (c >= W) return;
    int lo = 0, hi = cnt;          // first slot with token >= id
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sorted_tok[mid] < id) lo = mid + 1; else hi = mid;
    }
    float s = 0.f;
    bool any = false;
    for (int j = lo; j < cnt && sorted_tok[j] == id; ++j) {
        s += dh[(size_t)sorted_rows[j] * W + c];
        any = true;
    }
    float* o = dtab + (size_t)id * W + c;
    if (!accumulate) *o = s;
    else if (any) *o += s;
}
// d pos_emb[t] (+)= sum_b dh[b, t]; d start_token (+)= sum_b dh[b, 0]
__global__ void pos_reduce_kernel(const float* __restrict__ dh, int n, int P, int W, float* dpos, float* dstart, int accumulate) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)P * W) return;
    float s = 0.f;
    for (int b = 0; b < n; ++b) s += dh[(size_t)b * P * W + i];
    if (dpos) dpos[i] = accumulate ? dpos[i] + s : s;
    if (dstart && i < (size_t)W) dstart[i] = accumulate ? dstart[i] + s : s;
}

// ---- cross-entropy head: loss[m] = lse - logit[target]; logits -> w_m (softmax - onehot) in place -------------------
__global__ void __launch_bounds__(256) xent_kernel(float* logits, const long long* __restrict__ targets,
                                                   const float* __restrict__ w_row, float* loss, int bins) {
    __shared__ float red[8];
    const size_t m = blockIdx.x;
    float* z = logits + m * bins;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float mx = -INFINITY;
    for (int i = tid; i < bins; i += 256) mx = fmaxf(mx, z[i]);
    mx = jk::warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
    __syncthreads();
    float s = 0.f;
    for (int i = tid; i < bins; i += 256) s += expf(z[i] - mx);
    s = jk::warp_sum(s);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < 8; ++w) tot += red[w];
    const long long tgt = targets[m];
    const float lse = mx + logf(tot);
    const float zt = z[tgt];
    __syncthreads();
    const float wr = w_row[m], inv = 1.f / tot;
    for (int i = tid; i < bins; i += 256) z[i] = wr * (expf(z[i] - mx) * inv - (i == tgt ? 1.f : 0.f));
    if (tid == 0) loss[m] = lse - zt;
}

inline unsigned blocks_for(size_t cnt, int t = 256) { return (unsigned)((cnt + t - 1) / t); }

int linear(const float* x, const float* w, const float* b, float* y, int M, int N, int K, int w_nk, cudaStream_t s) {
    return jk_f32_linear(x, w, b, y, M, N, K, w_nk, (jk_stream_t)s);
}

int wgrad(const float* x, const float* dy, float* dw, float* db, int M, int K, int N, int accumulate, cudaStream_t s) {
    if (dw) {
        wgrad_kernel<<<dim3((N + 63) / 64, (K + 63) / 64), 256, 0, s>>>(x, dy, dw, M, K, N, accumulate);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    if (db) {
        colsum_kernel<<<(N + 31) / 32, 256, 0, s>>>(dy, nullptr, nullptr, db, nullptr, M, N, accumulate);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

// dX (+)= LayerNorm backward of dY at input x; dgamma / dbeta added when non-NULL
int ln_backward(const float* x, const float* gamma, const float* dy, float* dx, float* dg, float* dbeta, float* stats,
                int M, int W, int accumulate, cudaStream_t s) {
    ln_bwd_kernel<<<M, 256, 0, s>>>(x, gamma, dy, dx, stats, W, 1e-5f, accumulate);
    JK_CHECK_CUDA(cudaGetLastError());
    if (dg || dbeta) {
        colsum_kernel<<<(W + 31) / 32, 256, 0, s>>>(dy, x, stats, dbeta, dg, M, W, 1);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

size_t attn_smem_bytes(int dh, int rows) { return (size_t)(2 * dh + 2 * rows) * sizeof(float); }

}  // namespace

extern "C" int jk_f32_linear_wgrad(const float* x, const float* dy, float* dw, float* db, int M, int K, int N,
                                   int accumulate, jk_stream_t stream) {
    JK_REQUIRE(x && dy && (dw || db), "null argument");
    JK_REQUIRE(M >= 1 && K >= 1 && N >= 1, "empty product [%d x %d] . [%d x %d]", K, M, M, N);
    return wgrad(x, dy, dw, db, M, K, N, accumulate ? 1 : 0, (cudaStream_t)stream);
}

extern "C" int jk_f32_backward_workspace_floats(const jk_f32_args* a, size_t* out) {
    JK_REQUIRE(a && out, "null argument");
    const size_t M = (size_t)a->n * a->P, W = a->width, S = a->n_state, Mw = a->mlp_width;
    // xn0, x1, xn1, dx1 [M, W]; qkv, dqkv [M, 3S]; att, datt [M, S]; a, g [M, Mw]; lse, D [n, H, P]; LN stats [M, 2]
    size_t f = M * (4 * W + 6 * S + 2 * S + 2 * Mw) + 2 * (size_t)a->n * a->heads * a->P + 2 * M;
    if (a->encoder_dims > 0) {
        const size_t E = (size_t)a->n * a->encoder_dims;
        f += E * (2 * S > W ? 2 * S : W) + E * 2 * S;   // kv of c_enc_kv (later d_encoder_kv's product), its gradient
        f += E * S * 2;              // dK, dV of the encoder rows before the merge
    }
    *out = f;
    return 0;
}

extern "C" int jk_f32_backward(const jk_f32_args* a, const jk_f32_layer* layers, const jk_f32_grad_layer* grads,
                               const float* const* saved_inputs, float* dx, float* d_encoder_kv, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(a && layers && grads && saved_inputs && dx && a->work, "null argument");
    const int n = a->n, P = a->P, W = a->width, S = a->n_state, Mw = a->mlp_width, H = a->heads;
    JK_REQUIRE(n >= 1 && a->depth >= 1, "n %d, depth %d", n, a->depth);
    JK_REQUIRE(a->p0 == 0 && P == a->n_ctx, "the backward runs whole windows: positions [%d, %d) of a context of %d",
               a->p0, a->p0 + P, a->n_ctx);
    JK_REQUIRE(H >= 1 && S % H == 0, "n_state %% heads != 0");
    const int dh = S / H, M = n * P;
    const int bc = a->blocks > 0 ? a->n_ctx / a->blocks : a->n_ctx;
    const int prime = a->blocks > 0 ? (a->prime_len / a->blocks + 1) * a->blocks : 0;
    const int E = a->encoder_dims;
    // every layer is checked before the first launch: .grad is accumulated in place
    for (int l = 0; l < a->depth; ++l) {
        const jk_f32_layer& L = layers[l];
        const int af = L.attn_func;
        JK_REQUIRE(af == 0 || af == 1 || af == 2 || af == 3 || af == 6 || af == 7,
                   "layer %d: attn_func %d has no backward in the fp32 path", l, af);
        JK_REQUIRE(saved_inputs[l], "layer %d: its saved input is required", l);
        JK_REQUIRE(L.ln0_g && L.ln0_b && L.ln1_g && L.ln1_b && L.c_attn_w && L.c_attn_b && L.c_proj_w && L.c_proj_b &&
                   L.fc_w && L.fc_b && L.proj2_w && L.proj2_b, "layer %d: a parameter pointer is NULL", l);
        JK_REQUIRE(af != 6 || (L.c_enc_kv_w && L.c_enc_kv_b && a->encoder_kv && E > 0),
                   "layer %d: an enc-dec layer needs encoder_kv and c_enc_kv", l);
        JK_REQUIRE(af != 7 || a->blocks > 0, "layer %d: a prime layer needs blocks", l);
        JK_REQUIRE((af != 1 && af != 2 && af != 3) || (a->blocks > 0 && a->n_ctx % a->blocks == 0),
                   "layer %d: a block pattern needs blocks dividing n_ctx", l);
        const int keys = af == 6 ? E : P;
        JK_REQUIRE(attn_smem_bytes(dh, keys) <= 96 * 1024 && attn_smem_bytes(dh, P) <= 96 * 1024,
                   "layer %d: attention rows of %d keys / %d queries do not fit shared memory", l, keys, P);
    }
    if (int rc = jk::set_max_smem_once<attn_fwd_kernel>(96 * 1024)) return rc;
    if (int rc = jk::set_max_smem_once<attn_bwd_query_kernel>(96 * 1024)) return rc;
    if (int rc = jk::set_max_smem_once<attn_bwd_key_kernel>(96 * 1024)) return rc;

    float* xn0 = a->work;
    float* x1 = xn0 + (size_t)M * W;
    float* xn1 = x1 + (size_t)M * W;
    float* dx1 = xn1 + (size_t)M * W;
    float* qkv = dx1 + (size_t)M * W;
    float* dqkv = qkv + (size_t)M * 3 * S;
    float* att = dqkv + (size_t)M * 3 * S;
    float* datt = att + (size_t)M * S;
    float* pre = datt + (size_t)M * S;
    float* g = pre + (size_t)M * Mw;
    float* lse = g + (size_t)M * Mw;
    float* dd = lse + (size_t)n * H * P;
    float* stats = dd + (size_t)n * H * P;
    float* kv = stats + 2 * (size_t)M;
    float* dkv = kv + (E > 0 ? (size_t)n * E * (2 * S > W ? 2 * S : W) : 0);
    float* dk_enc = dkv + (E > 0 ? (size_t)n * E * 2 * S : 0);
    float* dv_enc = dk_enc + (E > 0 ? (size_t)n * E * S : 0);
    const double sc = 1.0 / sqrt(sqrt((double)dh));
    const float scale2 = (float)(sc * sc);
    const size_t MW = (size_t)M * W;

    for (int l = a->depth - 1; l >= 0; --l) {
        const jk_f32_layer& L = layers[l];
        const jk_f32_grad_layer& G = grads[l];
        const int af = L.attn_func;
        const float* x = saved_inputs[l];
        int rc;
        // ---- recompute the layer's forward from its input ----
        if ((rc = jk_layernorm_f32(x, L.ln0_g, L.ln0_b, xn0, M, W, 1e-5f, stream_))) return rc;
        AttnG A{};
        A.P = P; A.S = S; A.H = H; A.dh = dh; A.bc = bc; A.attn_func = af; A.prime = prime; A.scale2 = scale2;
        A.o = att; A.o_w = att; A.dout = datt; A.lse = lse; A.dd = dd;
        if (af == 6) {
            if ((rc = linear(xn0, L.c_attn_w, L.c_attn_b, qkv, M, S, W, 0, stream))) return rc;
            if ((rc = linear(a->encoder_kv, L.c_enc_kv_w, L.c_enc_kv_b, kv, n * E, 2 * S, W, 0, stream))) return rc;
            A.q = qkv; A.q_stride = S; A.k = kv; A.v = kv + S; A.kv_stride = 2 * S; A.Lk = E;
            A.dq = dqkv; A.dq_stride = S; A.dk = dk_enc; A.dv = dv_enc; A.dkv_stride = S;
        } else {
            if ((rc = linear(xn0, L.c_attn_w, L.c_attn_b, qkv, M, 3 * S, W, 0, stream))) return rc;
            A.q = qkv; A.q_stride = 3 * S; A.k = qkv + S; A.v = qkv + 2 * S; A.kv_stride = 3 * S; A.Lk = P;
            A.dq = dqkv; A.dq_stride = 3 * S; A.dk = dqkv + S; A.dv = dqkv + 2 * S; A.dkv_stride = 3 * S;
        }
        attn_fwd_kernel<<<dim3(P, H, n), 128, (size_t)(A.dh + A.Lk) * sizeof(float), stream>>>(A);
        JK_CHECK_CUDA(cudaGetLastError());
        if ((rc = linear(att, L.c_proj_w, L.c_proj_b, x1, M, W, S, 0, stream))) return rc;
        add_kernel<<<blocks_for(MW), 256, 0, stream>>>(x1, x, MW);                  // x1 = x + a
        JK_CHECK_CUDA(cudaGetLastError());
        if ((rc = jk_layernorm_f32(x1, L.ln1_g, L.ln1_b, xn1, M, W, 1e-5f, stream_))) return rc;
        if ((rc = linear(xn1, L.fc_w, L.fc_b, pre, M, Mw, W, 0, stream))) return rc;
        gelu_kernel<<<blocks_for((size_t)M * Mw), 256, 0, stream>>>(pre, g, (size_t)M * Mw);
        JK_CHECK_CUDA(cudaGetLastError());

        // ---- MLP: h = x1 + g . proj2 + b ----
        if ((rc = wgrad(g, dx, G.proj2_w, G.proj2_b, M, Mw, W, 1, stream))) return rc;
        if ((rc = linear(dx, L.proj2_w, nullptr, g, M, Mw, W, 1, stream))) return rc;          // dG (over g)
        gelu_bwd_kernel<<<blocks_for((size_t)M * Mw), 256, 0, stream>>>(pre, g, (size_t)M * Mw);   // dA
        JK_CHECK_CUDA(cudaGetLastError());
        if ((rc = wgrad(xn1, g, G.fc_w, G.fc_b, M, W, Mw, 1, stream))) return rc;
        if ((rc = linear(g, L.fc_w, nullptr, xn1, M, W, Mw, 1, stream))) return rc;            // dXn1 (over xn1)
        JK_CHECK_CUDA(cudaMemcpyAsync(dx1, dx, MW * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        if ((rc = ln_backward(x1, L.ln1_g, xn1, dx1, G.ln1_g, G.ln1_b, stats, M, W, 1, stream))) return rc;

        // ---- attention: x1 = x + att . c_proj + b ----
        if ((rc = wgrad(att, dx1, G.c_proj_w, G.c_proj_b, M, S, W, 1, stream))) return rc;
        if ((rc = linear(dx1, L.c_proj_w, nullptr, datt, M, S, W, 1, stream))) return rc;
        attn_bwd_query_kernel<<<dim3(P, H, n), 128, attn_smem_bytes(dh, A.Lk), stream>>>(A);
        JK_CHECK_CUDA(cudaGetLastError());
        attn_bwd_key_kernel<<<dim3(A.Lk, H, n), 128, attn_smem_bytes(dh, P), stream>>>(A);
        JK_CHECK_CUDA(cudaGetLastError());
        const int qw = af == 6 ? S : 3 * S;
        if ((rc = wgrad(xn0, dqkv, G.c_attn_w, G.c_attn_b, M, W, qw, 1, stream))) return rc;
        if ((rc = linear(dqkv, L.c_attn_w, nullptr, xn0, M, W, qw, 1, stream))) return rc;     // dXn0 (over xn0)
        if (af == 6 && (G.c_enc_kv_w || G.c_enc_kv_b || d_encoder_kv)) {
            const size_t rows = (size_t)n * E;
            merge_kv_kernel<<<blocks_for(rows * S), 256, 0, stream>>>(dk_enc, dv_enc, dkv, rows, S);
            JK_CHECK_CUDA(cudaGetLastError());
            if ((G.c_enc_kv_w || G.c_enc_kv_b) &&
                (rc = wgrad(a->encoder_kv, dkv, G.c_enc_kv_w, G.c_enc_kv_b, (int)rows, W, 2 * S, 1, stream))) return rc;
            if (d_encoder_kv) {
                if ((rc = linear(dkv, L.c_enc_kv_w, nullptr, kv, (int)rows, W, 2 * S, 1, stream))) return rc;
                add_kernel<<<blocks_for(rows * W), 256, 0, stream>>>(d_encoder_kv, kv, rows * W);
                JK_CHECK_CUDA(cudaGetLastError());
            }
        }
        // dx = dx1 + LN0 backward
        JK_CHECK_CUDA(cudaMemcpyAsync(dx, dx1, MW * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        if ((rc = ln_backward(x, L.ln0_g, xn0, dx, G.ln0_g, G.ln0_b, stats, M, W, 1, stream))) return rc;
    }
    return 0;
}

extern "C" int jk_f32_embed_backward(const float* dh, const int64_t* tokens, int64_t tok_stride, int n, int P, int width,
                                     int bins, float* d_x_emb, float* d_pos_emb, float* d_start_token, int* work,
                                     int accumulate, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(dh, "null argument");
    JK_REQUIRE(n >= 1 && P >= 1 && width >= 1, "n %d, P %d, width %d", n, P, width);
    JK_REQUIRE(!d_x_emb || P == 1 || (tokens && work && bins >= 1), "d_x_emb needs tokens, bins and the workspace");
    JK_REQUIRE((long long)n * P * bins < (1ll << 62), "too many rows");
    if (d_x_emb) {
        const int cnt = n * (P - 1);
        int* rows = work;
        int* tok = work + cnt;
        if (cnt > 0) {
            rank_sort_kernel<<<blocks_for(cnt), 256, 0, stream>>>((const long long*)tokens, tok_stride, n, P, rows, tok);
            JK_CHECK_CUDA(cudaGetLastError());
        }
        emb_reduce_kernel<<<dim3((width + 127) / 128, bins), 128, 0, stream>>>(dh, rows, tok, cnt, d_x_emb, bins, width,
                                                                                accumulate ? 1 : 0);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    if (d_pos_emb || d_start_token) {
        pos_reduce_kernel<<<blocks_for((size_t)P * width), 256, 0, stream>>>(dh, n, P, width, d_pos_emb, d_start_token,
                                                                             accumulate ? 1 : 0);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

extern "C" int jk_f32_xent_backward(float* logits, const int64_t* targets, const float* row_weight, float* loss, int M,
                                    int bins, jk_stream_t stream) {
    JK_REQUIRE(logits && targets && row_weight && loss, "null argument");
    JK_REQUIRE(M >= 1 && bins >= 1, "M %d, bins %d", M, bins);
    xent_kernel<<<M, 256, 0, (cudaStream_t)stream>>>(logits, (const long long*)targets, row_weight, loss, bins);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}
