// fp32 transformer path: Transformer.forward in fp32 - forward mode over a whole sequence (training-shaped / alignment,
// transformer/transformer.py:169-192 with sample=False, factored_attention.py:135-228 masks) and sampling mode with fp32
// K/V caches (ConditionalAutoregressive2D.sample(fp16=False), prior/autoregressive.py:199-249, as train.py:139 calls it).
//
// This is NOT the hot path (the reference samples in fp16, sample.py:239-241): the kernels here are plain fp32 CUDA-core
// code written for exactness against the reference's fp32 outputs (tests: golden `y32`, `yfull32`, `preds32` at 2e-5),
// one launch per operator, orchestrated per layer by jk_f32_forward.  All arithmetic is fp32 (no TF32):
//   LayerNorm (ops.py:14-24) -> Conv1D (ops.py:83-101) -> attention (factored_attention.py:82-108: scores scaled by
//   dh^-1/2, softmax, .v) over the key set of the layer's pattern -> Conv1D + residual -> LayerNorm -> Conv1D +
//   quick_gelu (ops.py:33-35) -> Conv1D + residual (transformer.py:82-83).
// Forward mode and sampling mode share ONE attention kernel: the keys of query position p are the cache rows the pattern
// attends (block: its block up to p; transpose: p - k*bc; previous block; prime: first _prime_len rows up to p; dense:
// all up to p; enc-dec: every encoder row) - forward mode simply runs with a cache that holds the whole sequence, which
// is what the reference's own check_sample asserts to be equal (factored_attention.py:424-455).
#include "common.cuh"
#include "../../include/jkb200.h"

namespace {

// ---- y[M, N] = epi(x[M, K] . w + b [, res]);  w is [K, N] (Conv1D layout) or [N, K] (nn.Linear layout, w_nk) ----------
// 64 x 64 output tile, K tile 16, 256 threads each 4 x 4 outputs.  fp32 FMAs.
enum { F32_EPI_NONE = 0, F32_EPI_GELU = 1, F32_EPI_RESIDUAL = 2 };

__global__ void __launch_bounds__(256) sgemm_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                     const float* __restrict__ b, const float* res, float* y, int M, int N, int K,
                                                     int w_nk, int epi) {
    __shared__ float xs[16][64 + 4];     // [k][m]
    __shared__ float ws[16][64 + 4];     // [k][n]
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < K; k0 += 16) {
        for (int i = tid; i < 64 * 16; i += 256) {
            const int m = i >> 4, k = i & 15;
            xs[k][m] = (m0 + m < M && k0 + k < K) ? x[(size_t)(m0 + m) * K + k0 + k] : 0.f;
        }
        if (w_nk) {
            for (int i = tid; i < 64 * 16; i += 256) {
                const int n = i >> 4, k = i & 15;
                ws[k][n] = (n0 + n < N && k0 + k < K) ? w[(size_t)(n0 + n) * K + k0 + k] : 0.f;
            }
        } else {
            for (int i = tid; i < 64 * 16; i += 256) {
                const int k = i >> 6, n = i & 63;
                ws[k][n] = (n0 + n < N && k0 + k < K) ? w[(size_t)(k0 + k) * N + n0 + n] : 0.f;
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            float a[4], c[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = xs[k][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) c[j] = ws[k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], c[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float v = acc[i][j] + (b ? b[n] : 0.f);
            if (epi == F32_EPI_GELU) v = v * (1.0f / (1.0f + expf(-1.702f * v)));
            else if (epi == F32_EPI_RESIDUAL) v += res[(size_t)m * N + n];
            y[(size_t)m * N + n] = v;
        }
    }
}

int sgemm(const float* x, const float* w, const float* b, const float* res, float* y, int M, int N, int K, int w_nk, int epi,
          cudaStream_t stream) {
    dim3 grid((N + 63) / 64, (M + 63) / 64);
    sgemm_kernel<<<grid, 256, 0, stream>>>(x, w, b, res, y, M, N, K, w_nk, epi);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---- K / V of the new positions -> cache rows (absolute positions) ------------------------------------------------
__global__ void kv_store_kernel(const float* __restrict__ qkv, float* kc, float* vc, int n, int P, int p0, int S, int Lc, int limit) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * P * S) return;
    const int s = (int)(i % S);
    const int m = (int)(i / S), b = m / P, p = p0 + m % P;
    if (p >= limit) return;                 // prime layers stop caching at _prime_len (factored_attention.py:255-271)
    const float* src = qkv + (size_t)m * 3 * S + s;
    kc[((size_t)b * Lc + p) * S + s] = src[S];
    vc[((size_t)b * Lc + p) * S + s] = src[2 * S];
}
__global__ void split_kv_kernel(const float* __restrict__ kv, float* kc, float* vc, size_t rows, int S) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * S) return;
    const size_t r = i / S;
    const int s = (int)(i % S);
    kc[i] = kv[r * 2 * S + s];
    vc[i] = kv[r * 2 * S + S + s];
}

// ---- attention of query position p over the key rows of its pattern ---------------------------------------------------
struct AttnF32 {
    const float* q;       // query rows: q[(b * P + i) * q_stride + h * dh]
    const float* kc;      // [n][Lc][S]
    const float* vc;
    float* out;           // [n * P][S]
    float* w_out;         // optional [n][H][P][Lk] attention weights, or NULL
    int P, p0, S, H, dh, bc, attn_func, prime, Lc, q_stride, Lk;
    float scale2;
};
__device__ __forceinline__ int f32_nkeys(const AttnF32& A, int p) {
    switch (A.attn_func) {
        case 0: return p + 1;
        case 1: return p % A.bc + 1;
        case 2: return p / A.bc + 1;
        case 3: return p >= A.bc ? A.bc : 0;
        case 6: return A.Lc;
        case 7: return p < A.prime ? p + 1 : A.prime;
    }
    return 0;
}
__device__ __forceinline__ int f32_key(const AttnF32& A, int p, int j) {
    switch (A.attn_func) {
        case 1: return p - p % A.bc + j;
        case 2: return p % A.bc + j * A.bc;
        case 3: return (p / A.bc - 1) * A.bc + j;
    }
    return j;   // 0, 6, 7
}

__global__ void __launch_bounds__(128) attn_f32_kernel(AttnF32 A) {
    extern __shared__ float fsm[];
    float* qs = fsm;                 // [dh]
    float* sc = fsm + A.dh;          // [nk]
    __shared__ float red[4];
    const int i = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int p = A.p0 + i;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dh = A.dh, S = A.S;
    const size_t row = (size_t)b * A.P + i;
    float* out = A.out + row * S + h * dh;
    const int nk = f32_nkeys(A, p);
    float* wrow = A.w_out ? A.w_out + (((size_t)b * A.H + h) * A.P + i) * A.Lk : nullptr;
    if (nk == 0) {      // previous-block attention inside the first block: zero keys / values -> output 0
        for (int d = tid; d < dh; d += 128) out[d] = 0.f;
        if (wrow)
            for (int j = tid; j < A.Lk; j += 128) wrow[j] = 0.f;
        return;
    }
    for (int d = tid; d < dh; d += 128) qs[d] = A.q[row * A.q_stride + h * dh + d];
    __syncthreads();
    const float* kb = A.kc + (size_t)b * A.Lc * S + h * dh;
    const float* vb = A.vc + (size_t)b * A.Lc * S + h * dh;
    for (int j = warp; j < nk; j += 4) {
        const float* k = kb + (size_t)f32_key(A, p, j) * S;
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
    if (wrow) {
        for (int j = tid; j < A.Lk; j += 128) wrow[j] = 0.f;
        __syncthreads();
        for (int j = tid; j < nk; j += 128) wrow[f32_key(A, p, j)] = sc[j] * inv;
    }
    for (int d = tid; d < dh; d += 128) {
        float o = 0.f;
        for (int j = 0; j < nk; ++j) o = fmaf(sc[j] * inv, vb[(size_t)f32_key(A, p, j) * S + d], o);
        out[d] = o;
    }
}

__global__ void embed_f32_kernel(float* __restrict__ x, const long long* __restrict__ tokens, long long tok_stride,
                                 const float* __restrict__ y_cond, const float* __restrict__ x_cond, long long x_cond_len,
                                 const float* __restrict__ x_emb, const float* __restrict__ pos_emb,
                                 const float* __restrict__ start_token, int n, int P, int p0, int W) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * P * W) return;
    const int col = (int)(i % W);
    const int m = (int)(i / W), b = m / P, t = p0 + m % P;
    float v;
    if (t == 0) v = y_cond ? y_cond[(size_t)b * W + col] : start_token[col];
    else v = x_emb[(size_t)tokens[(size_t)b * tok_stride + t - 1] * W + col];
    v += pos_emb[(size_t)t * W + col];
    if (x_cond) v += x_cond[((size_t)b * x_cond_len + (x_cond_len > 1 ? t : 0)) * W + col];
    x[i] = v;
}

}  // namespace

extern "C" int jk_f32_workspace_floats(const jk_f32_args* a, size_t* out) {
    JK_REQUIRE(a && out, "null argument");
    const size_t M = (size_t)a->n * a->P;
    size_t f = M * ((size_t)a->width + 3 * (size_t)a->n_state + a->n_state + a->mlp_width);
    if (a->encoder_dims > 0) f += (size_t)a->n * a->encoder_dims * 2 * a->n_state;      // c_enc_kv output before the split
    *out = f;
    return 0;
}

extern "C" int jk_f32_forward(const jk_f32_args* a, const jk_f32_layer* layers, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(a && layers && a->x && a->work, "null argument");
    const int n = a->n, P = a->P, W = a->width, S = a->n_state, Mw = a->mlp_width, H = a->heads;
    JK_REQUIRE(n >= 1 && P >= 1 && a->p0 >= 0 && a->p0 + P <= a->n_ctx, "positions [%d, %d) outside the context %d", a->p0, a->p0 + P, a->n_ctx);
    JK_REQUIRE(S % H == 0, "n_state %% heads != 0");
    const int dh = S / H, M = n * P;
    const int bc = a->blocks > 0 ? a->n_ctx / a->blocks : a->n_ctx;
    const int prime = a->blocks > 0 ? (a->prime_len / a->blocks + 1) * a->blocks : 0;
    float* xn = a->work;
    float* qkv = xn + (size_t)M * W;
    float* att = qkv + (size_t)M * 3 * S;
    float* g = att + (size_t)M * S;
    float* enc_tmp = g + (size_t)M * Mw;
    double sc = 1.0 / sqrt(sqrt((double)dh));
    const float scale2 = (float)(sc * sc);
    // every layer is checked before the first launch: x is rewritten in place, so a table that fails at layer l must
    // not leave layers 0 .. l-1 applied
    for (int l = 0; l < a->depth; ++l) {
        const jk_f32_layer& L = layers[l];
        const int af = L.attn_func;
        JK_REQUIRE(af == 0 || af == 1 || af == 2 || af == 3 || af == 6 || af == 7, "layer %d: attn_func %d is not built in the fp32 path", l, af);
        JK_REQUIRE(L.k_cache && L.v_cache, "layer %d: K/V cache (or forward-mode scratch) is required", l);
        JK_REQUIRE(af != 6 || a->encoder_kv || a->p0 > 0, "layer %d: encoder_kv is required at position 0", l);
        const int Lc = (af == 6) ? a->encoder_dims : a->n_ctx;
        JK_REQUIRE((size_t)(dh + Lc) * sizeof(float) <= 96 * 1024, "layer %d: attention row of %d keys does not fit shared memory in the fp32 path", l, Lc);
    }
    if (int rc = jk::set_max_smem_once<attn_f32_kernel>(96 * 1024)) return rc;
    for (int l = 0; l < a->depth; ++l) {
        const jk_f32_layer& L = layers[l];
        const int af = L.attn_func;
        int rc = jk_layernorm_f32(a->x, L.ln0_g, L.ln0_b, xn, M, W, 1e-5f, stream_);
        if (rc) return rc;
        const int Lc = (af == 6) ? a->encoder_dims : a->n_ctx;
        AttnF32 A;
        A.kc = L.k_cache; A.vc = L.v_cache; A.out = att; A.w_out = L.attn_w; A.P = P; A.p0 = a->p0; A.S = S; A.H = H; A.dh = dh;
        A.bc = bc; A.attn_func = af; A.prime = prime; A.Lc = Lc; A.Lk = Lc; A.scale2 = scale2;
        if (af == 6) {
            rc = sgemm(xn, L.c_attn_w, L.c_attn_b, nullptr, qkv, M, S, W, 0, F32_EPI_NONE, stream);
            if (rc) return rc;
            if (a->p0 == 0) {      // c_enc_kv(encoder_kv) once per window (factored_attention.py:273-287)
                const size_t rows = (size_t)n * a->encoder_dims;
                rc = sgemm(a->encoder_kv, L.c_enc_kv_w, L.c_enc_kv_b, nullptr, enc_tmp, (int)rows, 2 * S, W, 0, F32_EPI_NONE, stream);
                if (rc) return rc;
                split_kv_kernel<<<(unsigned)((rows * S + 255) / 256), 256, 0, stream>>>(enc_tmp, L.k_cache, L.v_cache, rows, S);
                JK_CHECK_CUDA(cudaGetLastError());
            }
            A.q = qkv; A.q_stride = S;
        } else {
            rc = sgemm(xn, L.c_attn_w, L.c_attn_b, nullptr, qkv, M, 3 * S, W, 0, F32_EPI_NONE, stream);
            if (rc) return rc;
            const size_t cnt = (size_t)M * S;
            kv_store_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, stream>>>(qkv, L.k_cache, L.v_cache, n, P, a->p0, S, Lc,
                                                                              af == 7 ? prime : a->n_ctx);
            JK_CHECK_CUDA(cudaGetLastError());
            A.q = qkv; A.q_stride = 3 * S;
        }
        const size_t smem = (size_t)(dh + Lc) * sizeof(float);
        attn_f32_kernel<<<dim3(P, H, n), 128, smem, stream>>>(A);
        JK_CHECK_CUDA(cudaGetLastError());
        rc = sgemm(att, L.c_proj_w, L.c_proj_b, a->x, a->x, M, W, S, 0, F32_EPI_RESIDUAL, stream);      // x1 = x + a
        if (rc) return rc;
        rc = jk_layernorm_f32(a->x, L.ln1_g, L.ln1_b, xn, M, W, 1e-5f, stream_);
        if (rc) return rc;
        rc = sgemm(xn, L.fc_w, L.fc_b, nullptr, g, M, Mw, W, 0, F32_EPI_GELU, stream);
        if (rc) return rc;
        rc = sgemm(g, L.proj2_w, L.proj2_b, a->x, a->x, M, W, Mw, 0, F32_EPI_RESIDUAL, stream);          // h = x1 + m
        if (rc) return rc;
    }
    return 0;
}

extern "C" int jk_f32_embed(float* x, const int64_t* tokens, int64_t tok_stride, const float* y_cond, const float* x_cond,
                            int64_t x_cond_len, const float* x_emb, const float* pos_emb, const float* start_token, int n, int P,
                            int p0, int width, jk_stream_t stream) {
    JK_REQUIRE(x && x_emb && pos_emb, "null argument");
    JK_REQUIRE(P >= 1 && (tokens || (p0 == 0 && P == 1)), "tokens required beyond position 0");
    JK_REQUIRE(y_cond || start_token || p0 > 0, "position 0 needs y_cond or the start token");
    const size_t cnt = (size_t)n * P * width;
    embed_f32_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, (const long long*)tokens, tok_stride, y_cond, x_cond,
                                                                                     x_cond_len ? x_cond_len : 1, x_emb, pos_emb,
                                                                                     start_token, n, P, p0, width);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_f32_linear(const float* x, const float* w, const float* b, float* y, int M, int N, int K, int w_is_nk,
                             jk_stream_t stream) {
    JK_REQUIRE(x && w && y, "null argument");
    return sgemm(x, w, b, nullptr, y, M, N, K, w_is_nk ? 1 : 0, F32_EPI_NONE, (cudaStream_t)stream);
}
