// Chunked prefill: all given (prime) positions of a window through every layer at once.
//
// Reference: ConditionalAutoregressive2D.primed_sample (prior/autoregressive.py:251-359) runs the given
// tokens through the transformer in chunks before sampling, and its own check (:330-338, check_chunks)
// asserts chunked == token-by-token.  The decode kernel (decode_engine.cu) is the token-by-token form; this
// file is the chunked form: M = n_samples x P rows per GEMM, so the four Conv1Ds of a layer run on the
// wgmma GEMM (prefill_gemm.cu) instead of streaming 1.8 GB of weights once per position.
//
// Per layer (rows m = b*P + p, fp16 activations, the decode kernel's rounding points):
//   xn  = LN0(x)                      ln_rows_kernel            (ops.py:14-24)
//   qkv = xn . Wqkv + b               gemm_f16_tc epi 0         (factored_attention.py:289-301)
//   a   = attention(q, K, V)          attn_fwd_kernel           (factored_attention.py:82-228, per pattern)
//   K, V -> the engine's caches       kv_scatter_kernel         (the layouts decode_engine.cu attends)
//   x1  = x + (a . Wo + b)            gemm_f16_tc epi 2         (transformer.py:82)
//   g   = quick_gelu(LN1(x1) . W1 + b)   ln_rows_kernel + gemm_f16_tc epi 1
//   x   = x1 + (g . W2 + b)           gemm_f16_tc epi 2         (transformer.py:83)
// Afterwards the engine stands at position P exactly as if P decode steps had run: only the K/V caches and
// the position carry over between steps.
//
// A continuation (engine at t0 > 0) runs positions t0 .. t0+P-1 on top of the rows' caches: row m = b*P + i is position
// t0 + i.  Its queries attend FROM the cache (the decode layout, where every pattern's keys are one run of rows), after
// the new K / V are scattered into it: the whole chunk first for the layouts with a row per position (0, 2, 7), block
// by block for the rings (1 keeps one block, 3 two), whose rows a later block of the chunk overwrites.
#include "engine.cuh"
#include <algorithm>

using namespace jk;

namespace {

__device__ __forceinline__ float ldh(const __half* p) { return __half2float(*p); }

// ---- embedding (autoregressive.py:177-197; decode_engine.cu phase P0) ---------------------------------
// row m = b*P + i is position t0 + i of sample b
__global__ void embed_rows_kernel(__half* __restrict__ x, const long long* __restrict__ tokens, long long tok_stride,
                                  const float* __restrict__ y_cond, const float* __restrict__ x_cond, long long x_cond_len,
                                  const float* __restrict__ x_emb, const float* __restrict__ pos_emb,
                                  const float* __restrict__ start_token, int n, int P, int t0, int W) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * P * W) return;
    const int col = (int)(i % W);
    const int m = (int)(i / W), b = m / P, t = t0 + m % P;
    float v;
    if (t == 0) v = y_cond ? y_cond[(size_t)b * W + col] : start_token[col];
    else v = x_emb[(size_t)tokens[(size_t)b * tok_stride + t - 1] * W + col];
    v += pos_emb[(size_t)t * W + col];
    if (x_cond) v += x_cond[((size_t)b * x_cond_len + (x_cond_len > 1 ? t : 0)) * W + col];
    x[i] = __float2half_rn(v);
}

// ---- LayerNorm of fp16 rows (fp32 math, eps 1e-5), one warp per row ------------------------------------
// same formulas as the decode kernel's staging: mean, var = E[x^2] - mean^2 (double for the cancellation),
// y = fp16(fma(fma(x, rstd, -mean*rstd), g, b))
__global__ void ln_rows_kernel(const __half* __restrict__ x, const float* __restrict__ g, const float* __restrict__ bta,
                               __half* __restrict__ y, int rows, int W) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const __half* xr = x + (size_t)row * W;
    double s1 = 0.0, s2 = 0.0;
    for (int c = lane * 8; c < W; c += 256) {
        const uint4 v = *reinterpret_cast<const uint4*>(xr + c);
        const __half* h = reinterpret_cast<const __half*>(&v);
#pragma unroll
        for (int e = 0; e < 8; ++e) { const float f = __half2float(h[e]); s1 += (double)f; s2 += (double)f * (double)f; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    const double rk = (double)(1.0f / (float)W);
    const double m = s1 * rk;
    double var = s2 * rk - m * m;
    var = var < 0.0 ? 0.0 : var;
    const float rstd = 1.0f / sqrtf((float)var + 1e-5f);
    const float nmr = -(float)m * rstd;
    for (int c = lane * 8; c < W; c += 256) {
        const uint4 v = *reinterpret_cast<const uint4*>(xr + c);
        const __half* h = reinterpret_cast<const __half*>(&v);
        __half o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e)
            o[e] = __float2half_rn(fmaf(fmaf(__half2float(h[e]), rstd, nmr), g[c + e], bta[c + e]));
        *reinterpret_cast<uint4*>(y + (size_t)row * W + c) = *reinterpret_cast<const uint4*>(o);
    }
}

// ---- attention, forward mode over the P given positions ------------------------------------------------
// One CTA per (position p, head h, sample b).  Keys of p by pattern (all inside [0, P)):
//   0 dense: 0..p     1 block: block start..p     2 transpose: p % bc + j*bc, j = 0..p/bc
//   3 previous block: (p/bc - 1)*bc .. +bc-1 (none in the first block -> output 0)     7 prime: 0..p (p < prime)
//   6 encoder-decoder: every encoder row; K / V come from the layer's cache (jk_prior_set_encoder_kv), q from c_attn
// Scores fp16(fp16(q.k) * dh^-1/2), softmax fp32, P rounded to fp16 (unnormalised), P.V fp32, / sum - the
// decode kernel's order of roundings.
// A continuation (cache = 1) runs queries at absolute positions: row i of qkv is position qoff + i, and this launch
// computes positions [qa, qb).  Its keys are read from the layer's K / V cache in the decode layout, where the keys of
// every pattern are one run of rows: key j of position p is cache row cache_row0(p) + j (decode_engine.cu attn_geom).
struct AttnFwd {
    const __half* qkv;   // [n*P][q_stride]: q | k | v per row (q only for an encoder-decoder layer)
    __half* a;           // [n*P][S]
    const __half *kc, *vc;   // the layer's K / V cache [n][H][rows][dhp] (encoder-decoder: rows = enc_rows)
    int P, S, H, dh, bc, attn_func, prime, q_stride, enc_rows, dhp;
    int qoff, qa, qb;    // position of qkv row 0 and the positions this launch computes (head of window: 0, 0, P)
    int cache, rows, blocks;   // keys from the cache (continuation), its rows per (sample, head), n_ctx / bc
    float scale2;
};

// the first cache row of position p's keys in the decode layout (attn_geom.base)
__device__ __forceinline__ int cache_row0(const AttnFwd& A, int p) {
    switch (A.attn_func) {
        case 2: return (p % A.bc) * A.blocks;
        case 3: return ((p / A.bc + 1) & 1) * A.bc;
    }
    return 0;   // 0, 1, 6, 7
}
// keys any position of [qa, qb) reads (shared memory of the scalar kernels)
__host__ __device__ __forceinline__ int fwd_max_keys(const AttnFwd& A) {
    const int k = A.cache ? A.qb : A.P;
    return k > A.enc_rows ? k : A.enc_rows;
}

__device__ __forceinline__ int fwd_nkeys(const AttnFwd& A, int p) {
    switch (A.attn_func) {
        case 0: return p + 1;
        case 1: return p % A.bc + 1;
        case 2: return p / A.bc + 1;
        case 3: return p >= A.bc ? A.bc : 0;
        case 6: return A.enc_rows;
        case 7: return p < A.prime ? p + 1 : A.prime;
    }
    return 0;
}
__device__ __forceinline__ int fwd_key(const AttnFwd& A, int p, int j) {
    if (A.cache) return cache_row0(A, p) + j;
    switch (A.attn_func) {
        case 1: return p - p % A.bc + j;
        case 2: return p % A.bc + j * A.bc;
        case 3: return (p / A.bc - 1) * A.bc + j;
    }
    return j;   // 0, 7
}

constexpr int kFwdThreads = 128;

// K / V rows of head h of sample b: key j of the pattern is row fwd_key(.., j) of kbase / vbase, `kstride` halfs apart
struct FwdKV {
    const __half* kbase;
    const __half* vbase;
    size_t kstride;
};
__device__ __forceinline__ FwdKV fwd_kv(const AttnFwd& A, int h, int b) {
    const bool enc = A.attn_func == 6, cached = enc || A.cache;
    const int S = A.S;
    const size_t cbase = ((size_t)b * A.H + h) * (enc ? A.enc_rows : A.rows) * A.dhp;
    FwdKV R;
    R.kbase = cached ? A.kc + cbase : A.qkv + (size_t)b * A.P * 3 * S + S + h * A.dh;
    R.vbase = cached ? A.vc + cbase : R.kbase + S;
    R.kstride = cached ? (size_t)A.dhp : (size_t)3 * S;
    return R;
}

// scores of query p over its nk > 0 keys -> sc[j], fp16(fp16(q.k) * dh^-1/2); returns the row max (one CTA of kFwdThreads)
__device__ __forceinline__ float fwd_row_scores(const AttnFwd& A, const FwdKV& R, int p, int h, int b, int nk, float* qs,
                                                float* sc, float* red) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dh = A.dh;
    const __half* q = A.qkv + ((size_t)b * A.P + (p - A.qoff)) * A.q_stride + h * dh;
    for (int d = tid; d < dh; d += kFwdThreads) qs[d] = ldh(q + d);
    __syncthreads();
    for (int j = warp; j < nk; j += kFwdThreads / 32) {
        const __half* k = R.kbase + (size_t)fwd_key(A, p, j) * R.kstride;
        float dot = 0.f;
        for (int d = lane; d < dh; d += 32) dot = fmaf(qs[d], ldh(k + d), dot);
        dot = warp_sum(dot);
        if (lane == 0) sc[j] = h2f_round(h2f_round(dot) * A.scale2);
    }
    __syncthreads();
    float mx = -INFINITY;
    for (int j = tid; j < nk; j += kFwdThreads) mx = fmaxf(mx, sc[j]);
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    __syncthreads();
    return mx;
}

__global__ void __launch_bounds__(kFwdThreads) attn_fwd_kernel(AttnFwd A) {
    extern __shared__ float fsm[];
    float* qs = fsm;                 // [dh]
    float* sc = fsm + A.dh;          // [nk]
    __shared__ float red[kFwdThreads / 32];
    const int p = A.qa + blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dh = A.dh, S = A.S;
    __half* out = A.a + ((size_t)b * A.P + (p - A.qoff)) * S + h * dh;
    const FwdKV R = fwd_kv(A, h, b);
    const int nk = fwd_nkeys(A, p);
    if (nk == 0) {
        for (int d = tid; d < dh; d += kFwdThreads) out[d] = __float2half_rn(0.f);
        return;
    }
    const float mx = fwd_row_scores(A, R, p, h, b, nk, qs, sc, red);
    float l = 0.f;
    for (int j = tid; j < nk; j += kFwdThreads) {
        const float e = expf(sc[j] - mx);
        l += e;
        sc[j] = h2f_round(e);
    }
    l = warp_sum(l);
    if (lane == 0) red[warp] = l;
    __syncthreads();
    const float inv = 1.f / (red[0] + red[1] + red[2] + red[3]);
    for (int d = tid; d < dh; d += kFwdThreads) {
        float o = 0.f;
        for (int j = 0; j < nk; ++j) {
            o = fmaf(sc[j], ldh(R.vbase + (size_t)fwd_key(A, p, j) * R.kstride + d), o);
        }
        out[d] = __float2half_rn(o * inv);
    }
}

// recorded weights of query p (see attn_record_mma_kernel) for the head geometries the tensor-core kernels do not take
// (dh > 256: the released upsamplers' 480): w[b][h][p][key] = fp16(exp(s - max) / sum) for keys < ld
__global__ void __launch_bounds__(kFwdThreads) attn_record_kernel(AttnFwd A, __half* __restrict__ w, int ld) {
    extern __shared__ float fsm[];
    float* qs = fsm;                 // [dh]
    float* sc = fsm + A.dh;          // [nk]
    __shared__ float red[kFwdThreads / 32];
    const int p = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nk = fwd_nkeys(A, p);
    if (nk == 0) return;             // a row without keys stays as the caller zeroed it
    const float mx = fwd_row_scores(A, fwd_kv(A, h, b), p, h, b, nk, qs, sc, red);
    float l = 0.f;
    for (int j = tid; j < nk; j += kFwdThreads) l += expf(sc[j] - mx);
    l = warp_sum(l);
    if (lane == 0) red[warp] = l;
    __syncthreads();
    const float inv = 1.f / (red[0] + red[1] + red[2] + red[3]);
    __half* wrow = w + (((size_t)b * A.H + h) * A.P + p) * ld;
    for (int j = tid; j < nk; j += kFwdThreads) {
        const int k = fwd_key(A, p, j);
        if (k < ld) wrow[k] = __float2half_rn(expf(sc[j] - mx) * inv);
    }
}

// ---- the same attention on the tensor cores (mma.sync.m16n8k16), flash style --------------------------------
// Every pattern is a set of independent SEQUENCES: queries q_pos(i) = q0 + i*qs (i < nq) attend keys k_pos(j) = k0 + j*ks
// (j < nk) with k_pos <= q_pos:
//   block: one sequence per block (q = k = the block's rows)       transpose: one per residue r (rows r, r+bc, ...)
//   previous block: q = block s, k = block s-1 (none for s = 0)    dense: one sequence of all rows
//   prime: q = all rows, k = the first min(prime, P) rows          encoder-decoder: q = all rows, k = every cache row (no mask)
// so that QK^T and PV are dense [64 x dh].[dh x 32] / [64 x 32].[32 x dh] tiles.  One CTA = 64 queries of one (sequence,
// head, sample): 4 warps x 16 query rows, Q fragments in registers, K / V tiles of 32 keys staged with cp.async (gathered
// rows), online softmax in fp32 with the decode kernel's roundings (score = fp16(fp16(q.k) * dh^-1/2); P rounded to fp16
// for P.V, the row sum kept in fp32 from the unrounded exponentials).  dh <= DH (zero padded), dh even.
// A continuation (AttnFwd.cache) has the same sequences over the absolute positions [qa, qb): one per block (1, 3) or
// residue (2) the range touches, else one; its keys are the cache rows krow0 + j (every pattern's keys are one run of
// cache rows) and start at position 0 of the window, not of the call.
struct AttnSeqs {
    int attn_func, bc, P, prime, enc_rows, tiles_per_seq;
    int cache, qa, qb, blocks;
};
struct SeqGeom { int q0, qs, nq, k0, ks, nk, krow0; };
__device__ __forceinline__ SeqGeom seq_geom_cache(const AttnSeqs& Q, int s) {
    SeqGeom g;
    g.qs = 1; g.ks = 1; g.k0 = 0; g.krow0 = 0; g.q0 = Q.qa; g.nq = Q.qb - Q.qa;
    const int bc = Q.bc;
    switch (Q.attn_func) {
        case 1: case 3: {
            const int sb = Q.qa / bc + s;                  // the block of this sequence
            g.q0 = max(Q.qa, sb * bc); g.nq = max(0, min(Q.qb, (sb + 1) * bc) - g.q0);
            if (Q.attn_func == 1) { g.k0 = sb * bc; g.nk = g.nq ? g.q0 + g.nq - g.k0 : 0; }
            else { g.k0 = (sb - 1) * bc; g.nk = sb ? bc : 0; g.krow0 = ((sb + 1) & 1) * bc; }
            break;
        }
        case 2: {
            g.q0 = Q.qa + s; g.qs = bc; g.nq = g.q0 < Q.qb ? (Q.qb - g.q0 + bc - 1) / bc : 0;
            const int r = g.q0 % bc;
            g.k0 = r; g.ks = bc; g.nk = g.nq ? (g.q0 - r) / bc + g.nq : 0; g.krow0 = r * Q.blocks;
            break;
        }
        case 6: g.nk = Q.enc_rows; break;
        case 7: g.nk = min(Q.prime, Q.qb); break;
        default: g.nk = Q.qb; break;
    }
    return g;
}
__device__ __forceinline__ SeqGeom seq_geom(const AttnSeqs& Q, int s) {
    if (Q.cache) return seq_geom_cache(Q, s);
    SeqGeom g;
    g.krow0 = 0;
    switch (Q.attn_func) {
        case 1: g.q0 = s * Q.bc; g.qs = 1; g.nq = min(Q.bc, Q.P - g.q0); g.k0 = g.q0; g.ks = 1; g.nk = g.nq; break;
        case 2: g.q0 = s; g.qs = Q.bc; g.nq = s < Q.P ? (Q.P - s + Q.bc - 1) / Q.bc : 0; g.k0 = s; g.ks = Q.bc; g.nk = g.nq; break;
        case 3: g.q0 = s * Q.bc; g.qs = 1; g.nq = min(Q.bc, Q.P - g.q0); g.k0 = (s - 1) * Q.bc; g.ks = 1; g.nk = s ? Q.bc : 0; break;
        case 6: g.q0 = 0; g.qs = 1; g.nq = Q.P; g.k0 = 0; g.ks = 1; g.nk = Q.enc_rows; break;
        case 7: g.q0 = 0; g.qs = 1; g.nq = Q.P; g.k0 = 0; g.ks = 1; g.nk = min(Q.prime, Q.P); break;
        default: g.q0 = 0; g.qs = 1; g.nq = Q.P; g.k0 = 0; g.ks = 1; g.nk = Q.P; break;
    }
    return g;
}

__device__ __forceinline__ void cp16(void* smem, const void* gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void ldsm_t4(uint32_t (&r)[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// Pieces of the tensor-core attention shared by the forward kernel and the record kernel below.
// W16: head rows are 16-byte aligned (dh % 8 == 0) -> 16-byte cp.async chunks; else (5b_lyrics: dh 150) 4-byte words
constexpr int kBQ = 64, kBK = 32;

// the tile of 64 queries i0.. of one sequence -> shared memory (zero rows / columns beyond nq / dh) -> this warp's A fragments
template <int DH, bool W16>
__device__ __forceinline__ void load_q_frags(uint32_t (&qf)[DH / 16][4], __half* qs, const AttnFwd& A, const SeqGeom& G,
                                             long long rowbase, int i0, int h) {
    constexpr int XS = DH + 8;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dh = A.dh, nv = dh >> 3;                       // 16-byte chunks per row
    if (W16) {
        for (int i = tid; i < kBQ * (DH / 8); i += 128) {
            const int r = i / (DH / 8), c = i % (DH / 8);
            uint4 v = make_uint4(0, 0, 0, 0);
            if (i0 + r < G.nq && c < nv)
                v = *reinterpret_cast<const uint4*>(A.qkv + (size_t)(rowbase + G.q0 + (long long)(i0 + r) * G.qs) * A.q_stride + h * dh + c * 8);
            *reinterpret_cast<uint4*>(qs + r * XS + c * 8) = v;
        }
    } else {
        for (int i = tid; i < kBQ * (DH / 2); i += 128) {
            const int r = i / (DH / 2), c = i % (DH / 2);
            uint32_t v = 0;
            if (i0 + r < G.nq && 2 * c < dh)
                v = *reinterpret_cast<const uint32_t*>(A.qkv + (size_t)(rowbase + G.q0 + (long long)(i0 + r) * G.qs) * A.q_stride + h * dh + c * 2);
            *reinterpret_cast<uint32_t*>(qs + r * XS + c * 2) = v;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < DH / 16; ++k) ldmatrix_x4(qf[k], qs + (warp * 16 + (lane & 15)) * XS + k * 16 + (lane >> 4) * 8);
}

// the keys a tile of queries attends: K / V rows kbase + j * kstride, j < nk
struct KeyRange {
    const __half* kbase;
    const __half* vbase;
    size_t kstride;
    int nk;
};
__device__ __forceinline__ KeyRange key_range(const AttnFwd& A, const SeqGeom& G, long long rowbase, int i0, int h, int b, bool enc) {
    KeyRange R;
    // keys beyond the last query of this tile are never needed
    int nk = G.nk;
    if (!enc && nk > 0) {
        const long long qmax = G.q0 + (long long)(min(i0 + kBQ, G.nq) - 1) * G.qs;
        const long long jm = qmax >= G.k0 ? (qmax - G.k0) / G.ks + 1 : 0;
        nk = (int)min((long long)nk, jm);
    }
    const int S = A.S;
    if (enc || A.cache) {        // cache rows krow0 + j
        const size_t base = (((size_t)b * A.H + h) * (enc ? A.enc_rows : A.rows) + G.krow0) * A.dhp;
        R.kbase = A.kc + base; R.vbase = A.vc + base;
        R.kstride = (size_t)A.dhp;
    } else {
        R.kbase = A.qkv + (size_t)(rowbase + (nk > 0 ? G.k0 : 0)) * 3 * S + S + h * A.dh; R.vbase = R.kbase + S;
        R.kstride = (size_t)3 * S * G.ks;
    }
    R.nk = nk;
    return R;
}

// keys j0 .. j0 + 31 (and their values when KV) -> shared memory; rows beyond nk and columns beyond dh are zero
template <int DH, bool W16, bool KV>
__device__ __forceinline__ void stage_keys(__half* ks, __half* vs, const KeyRange& R, int j0, int dh) {
    constexpr int XS = DH + 8;
    const int tid = threadIdx.x, nv = dh >> 3;
    if (W16) {
        for (int i = tid; i < kBK * (DH / 8); i += 128) {
            const int r = i / (DH / 8), c = i % (DH / 8);
            if (j0 + r < R.nk && c < nv) {
                cp16(ks + r * XS + c * 8, R.kbase + (size_t)(j0 + r) * R.kstride + c * 8);
                if (KV) cp16(vs + r * XS + c * 8, R.vbase + (size_t)(j0 + r) * R.kstride + c * 8);
            } else {
                *reinterpret_cast<uint4*>(ks + r * XS + c * 8) = make_uint4(0, 0, 0, 0);
                if (KV) *reinterpret_cast<uint4*>(vs + r * XS + c * 8) = make_uint4(0, 0, 0, 0);
            }
        }
        asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
    } else {
#pragma unroll 4
        for (int i = tid; i < kBK * (DH / 2); i += 128) {
            const int r = i / (DH / 2), c = i % (DH / 2);
            uint32_t kv = 0, vv = 0;
            if (j0 + r < R.nk && 2 * c < dh) {
                kv = *reinterpret_cast<const uint32_t*>(R.kbase + (size_t)(j0 + r) * R.kstride + c * 2);
                if (KV) vv = *reinterpret_cast<const uint32_t*>(R.vbase + (size_t)(j0 + r) * R.kstride + c * 2);
            }
            *reinterpret_cast<uint32_t*>(ks + r * XS + c * 2) = kv;
            if (KV) *reinterpret_cast<uint32_t*>(vs + r * XS + c * 2) = vv;
        }
    }
}

// S = Q K^T of this warp's 16 query rows x the 32 staged keys, with the reference's roundings
// (score = fp16(fp16(q.k) * dh^-1/2)); keys outside the pattern (j >= nk, or after the query) are -inf.
// sc[n][e]: key j0 + n*8 + 2*t4 + (e & 1) of query row qp0 (e < 2) or qp1 (e >= 2)
template <int DH>
__device__ __forceinline__ void tile_scores(float (&sc)[kBK / 8][4], const uint32_t (&qf)[DH / 16][4], const __half* ks,
                                            const SeqGeom& G, int j0, int nk, long long qp0, long long qp1, bool enc, float scale2) {
    constexpr int XS = DH + 8;
    const int lane = threadIdx.x & 31, t4 = lane & 3;
#pragma unroll
    for (int n = 0; n < kBK / 8; ++n) sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
#pragma unroll
    for (int k = 0; k < DH / 16; ++k) {
#pragma unroll
        for (int np = 0; np < kBK / 16; ++np) {
            uint32_t kf[4];
            ldmatrix_x4(kf, ks + (np * 16 + (lane & 7) + ((lane >> 4) << 3)) * XS + k * 16 + ((lane >> 3) & 1) * 8);
            mma_16816(sc[2 * np], qf[k], kf[0], kf[1]);
            mma_16816(sc[2 * np + 1], qf[k], kf[2], kf[3]);
        }
    }
#pragma unroll
    for (int n = 0; n < kBK / 8; ++n)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int j = j0 + n * 8 + 2 * t4 + (e & 1);
            const long long kp = G.k0 + (long long)j * G.ks;
            const bool ok = j < nk && (enc || kp <= (e >= 2 ? qp1 : qp0));
            sc[n][e] = ok ? h2f_round(h2f_round(sc[n][e]) * scale2) : -INFINITY;
        }
}

// the running row max / row sum (fp32, from the unrounded exponentials) of quad-shared rows after one tile of scores;
// returns the rescale factors of the previous sums
__device__ __forceinline__ void online_max(const float (&sc)[kBK / 8][4], float& m0, float& m1, float& c0, float& c1) {
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int n = 0; n < kBK / 8; ++n)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            if (e >= 2) mx1 = fmaxf(mx1, sc[n][e]); else mx0 = fmaxf(mx0, sc[n][e]);
        }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    c0 = expf(m0 - mx0); c1 = expf(m1 - mx1);
    m0 = mx0; m1 = mx1;
}

template <int DH, bool W16>
__global__ void __launch_bounds__(128) attn_fwd_mma_kernel(AttnFwd A, AttnSeqs Q) {
    constexpr int XS = DH + 8, BQ = kBQ, BK = kBK;
    extern __shared__ __align__(16) __half asm_[];
    __half* qs = asm_;                       // [BQ][XS]
    __half* ks = qs + BQ * XS;               // [BK][XS]
    __half* vs = ks + BK * XS;               // [BK][XS]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t4 = lane & 3;
    const int seq = blockIdx.x / Q.tiles_per_seq, qt = blockIdx.x - seq * Q.tiles_per_seq;
    const int h = blockIdx.y, b = blockIdx.z;
    const SeqGeom G = seq_geom(Q, seq);
    const int i0 = qt * BQ;
    if (i0 >= G.nq) return;
    const int dh = A.dh, S = A.S;
    const bool enc = A.attn_func == 6;
    const long long rowbase = (long long)b * A.P - A.qoff;     // qkv row of position 0
    uint32_t qf[DH / 16][4];
    load_q_frags<DH, W16>(qf, qs, A, G, rowbase, i0, h);
    float o[DH / 8][4];
#pragma unroll
    for (int n = 0; n < DH / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float m0 = -1e30f, m1 = -1e30f, l0 = 0.f, l1 = 0.f;
    const int qi0 = i0 + warp * 16 + g, qi1 = qi0 + 8;                  // this lane's two query rows (sequence indices)
    const long long qp0 = G.q0 + (long long)qi0 * G.qs, qp1 = G.q0 + (long long)qi1 * G.qs;
    const KeyRange R = key_range(A, G, rowbase, i0, h, b, enc);
    for (int j0 = 0; j0 < R.nk; j0 += BK) {
        __syncthreads();                                                // the previous tile's fragment reads are done
        stage_keys<DH, W16, true>(ks, vs, R, j0, dh);
        __syncthreads();
        float sc[BK / 8][4];
        tile_scores<DH>(sc, qf, ks, G, j0, R.nk, qp0, qp1, enc, A.scale2);
        // ---- online softmax ----
        float c0, c1;
        online_max(sc, m0, m1, c0, c1);
        float r0 = 0.f, r1 = 0.f;
        uint32_t pf[BK / 16][4];
#pragma unroll
        for (int n = 0; n < BK / 8; ++n) {
            const float e0 = expf(sc[n][0] - m0), e1 = expf(sc[n][1] - m0), e2 = expf(sc[n][2] - m1), e3 = expf(sc[n][3] - m1);
            r0 += e0 + e1; r1 += e2 + e3;
            pf[n >> 1][(n & 1) * 2] = pack_h2(e0, e1);
            pf[n >> 1][(n & 1) * 2 + 1] = pack_h2(e2, e3);
        }
        r0 += __shfl_xor_sync(0xffffffffu, r0, 1); r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
        r1 += __shfl_xor_sync(0xffffffffu, r1, 1); r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
        l0 = l0 * c0 + r0; l1 = l1 * c1 + r1;
#pragma unroll
        for (int n = 0; n < DH / 8; ++n) { o[n][0] *= c0; o[n][1] *= c0; o[n][2] *= c1; o[n][3] *= c1; }
        // ---- O += P V ----
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) {
#pragma unroll
            for (int np = 0; np < DH / 16; ++np) {
                uint32_t vf[4];
                ldsm_t4(vf, vs + (kk * 16 + (lane & 15)) * XS + np * 16 + (lane >> 4) * 8);
                mma_16816(o[2 * np], pf[kk], vf[0], vf[1]);
                mma_16816(o[2 * np + 1], pf[kk], vf[2], vf[3]);
            }
        }
    }
    // ---- out = O / l (a row without keys - previous-block attention inside the first block - is 0) ----
    const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
#pragma unroll
    for (int n = 0; n < DH / 8; ++n) {
        const int d = n * 8 + 2 * t4;
        if (d < dh) {
            if (qi0 < G.nq) *reinterpret_cast<uint32_t*>(A.a + (size_t)(rowbase + qp0) * S + h * dh + d) = pack_h2(o[n][0] * inv0, o[n][1] * inv0);
            if (qi1 < G.nq) *reinterpret_cast<uint32_t*>(A.a + (size_t)(rowbase + qp1) * S + h * dh + d) = pack_h2(o[n][2] * inv1, o[n][3] * inv1);
        }
    }
}

// ---- recorded attention weights (record_attn, factored_attention.py:83-105 in fp16 mode) ----------------------------------
// w[b][h][q][k] = fp16(softmax_fp32(score)[k]) for every key k < ld of the query's pattern, score as above.  The weights are
// normalised BEFORE the fp16 rounding, so the forward kernel's unnormalised P cannot serve: the same tiles and key staging
// run twice, the first pass for the row max and row sum, the second for the write.  Entries outside the pattern are
// zeroed by the caller (cudaMemsetAsync), and so are rows without keys.
template <int DH, bool W16>
__global__ void __launch_bounds__(128) attn_record_mma_kernel(AttnFwd A, AttnSeqs Q, __half* __restrict__ w, int ld) {
    constexpr int XS = DH + 8;
    extern __shared__ __align__(16) __half asm_[];
    __half* qs = asm_;                       // [kBQ][XS]
    __half* ks = qs + kBQ * XS;              // [kBK][XS]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t4 = lane & 3;
    const int seq = blockIdx.x / Q.tiles_per_seq, qt = blockIdx.x - seq * Q.tiles_per_seq;
    const int h = blockIdx.y, b = blockIdx.z;
    const SeqGeom G = seq_geom(Q, seq);
    const int i0 = qt * kBQ;
    if (i0 >= G.nq) return;
    const bool enc = A.attn_func == 6;
    const long long rowbase = (long long)b * A.P - A.qoff;     // qkv row of position 0
    uint32_t qf[DH / 16][4];
    load_q_frags<DH, W16>(qf, qs, A, G, rowbase, i0, h);
    const int qi0 = i0 + warp * 16 + g, qi1 = qi0 + 8;
    const long long qp0 = G.q0 + (long long)qi0 * G.qs, qp1 = G.q0 + (long long)qi1 * G.qs;
    const KeyRange R = key_range(A, G, rowbase, i0, h, b, enc);
    // ---- pass 1: row max and row sum ----
    float m0 = -1e30f, m1 = -1e30f, l0 = 0.f, l1 = 0.f;
    for (int j0 = 0; j0 < R.nk; j0 += kBK) {
        __syncthreads();
        stage_keys<DH, W16, false>(ks, nullptr, R, j0, A.dh);
        __syncthreads();
        float sc[kBK / 8][4];
        tile_scores<DH>(sc, qf, ks, G, j0, R.nk, qp0, qp1, enc, A.scale2);
        float c0, c1;
        online_max(sc, m0, m1, c0, c1);
        float r0 = 0.f, r1 = 0.f;
#pragma unroll
        for (int n = 0; n < kBK / 8; ++n) {
            r0 += expf(sc[n][0] - m0) + expf(sc[n][1] - m0);
            r1 += expf(sc[n][2] - m1) + expf(sc[n][3] - m1);
        }
        r0 += __shfl_xor_sync(0xffffffffu, r0, 1); r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
        r1 += __shfl_xor_sync(0xffffffffu, r1, 1); r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
        l0 = l0 * c0 + r0; l1 = l1 * c1 + r1;
    }
    // ---- pass 2: fp16(exp(s - max) / sum) of the keys below ld ----
    const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
    __half* w0 = w + (((size_t)b * A.H + h) * A.P + (size_t)qp0) * ld;
    __half* w1 = w + (((size_t)b * A.H + h) * A.P + (size_t)qp1) * ld;
    for (int j0 = 0; j0 < R.nk && G.k0 + (long long)j0 * G.ks < ld; j0 += kBK) {
        __syncthreads();
        stage_keys<DH, W16, false>(ks, nullptr, R, j0, A.dh);
        __syncthreads();
        float sc[kBK / 8][4];
        tile_scores<DH>(sc, qf, ks, G, j0, R.nk, qp0, qp1, enc, A.scale2);
#pragma unroll
        for (int n = 0; n < kBK / 8; ++n)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const bool row1 = e >= 2;
                const long long kp = G.k0 + (long long)(j0 + n * 8 + 2 * t4 + (e & 1)) * G.ks;
                if ((row1 ? qi1 : qi0) < G.nq && kp < ld && sc[n][e] != -INFINITY)
                    (row1 ? w1 : w0)[kp] = __float2half_rn(expf(sc[n][e] - (row1 ? m1 : m0)) * (row1 ? inv1 : inv0));
            }
    }
}

// w == nullptr: the forward (attn_fwd_mma_kernel); else the recorded weights of the layer (attn_record_mma_kernel)
template <int DH, bool W16>
int launch_attn_mma(const AttnFwd& A, const AttnSeqs& Q, int nseq, int n, __half* w, int ld, cudaStream_t stream) {
    const dim3 grid((unsigned)(nseq * Q.tiles_per_seq), A.H, n);
    if (!w) {
        constexpr size_t smem = (size_t)(kBQ + 2 * kBK) * (DH + 8) * 2;
        if (int rc = set_max_smem_once<attn_fwd_mma_kernel<DH, W16>>((int)smem)) return rc;
        attn_fwd_mma_kernel<DH, W16><<<grid, 128, smem, stream>>>(A, Q);
    } else {
        constexpr size_t smem = (size_t)(kBQ + kBK) * (DH + 8) * 2;
        if (int rc = set_max_smem_once<attn_record_mma_kernel<DH, W16>>((int)smem)) return rc;
        attn_record_mma_kernel<DH, W16><<<grid, 128, smem, stream>>>(A, Q, w, ld);
    }
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// the kernels that take a layer's attention: the tensor-core kernels for even dh <= 256 (16-byte staging when every head
// row is 16-byte aligned, 4-byte words otherwise), the scalar kernels for other head sizes or when `scalar` asks for them
jk_prefill_attn_route attn_route(const AttnFwd& A, bool scalar) {
    jk_prefill_attn_route r = {0, 0, 0};
    if (scalar || A.dh % 2 != 0 || A.dh > 256) return r;
    const bool w16 = A.dh % 8 == 0 && A.S % 8 == 0 && A.dhp % 8 == 0;
    r.tensor_cores = 1;
    r.stage_bytes = w16 ? 16 : 4;
    r.tile_dh = !w16 ? (A.dh <= 160 ? 160 : 256) : A.dh <= 32 ? 32 : A.dh <= 64 ? 64 : A.dh <= 128 ? 128 : 256;
    return r;
}

// the layer's attention (w == nullptr) or its recorded weights on the tensor cores, route r (attn_route, tensor_cores 1)
int attn_mma(const AttnFwd& A, const jk_prefill_attn_route& r, int n, __half* w, int ld, cudaStream_t stream) {
    AttnSeqs Q;
    Q.attn_func = A.attn_func; Q.bc = A.bc; Q.P = A.P; Q.prime = A.prime; Q.enc_rows = A.enc_rows;
    Q.cache = A.cache; Q.qa = A.qa; Q.qb = A.qb; Q.blocks = A.blocks;
    const int nq = A.qb - A.qa;          // the head of a window: P
    int nseq = 1, maxq = nq;
    switch (A.attn_func) {
        case 1: case 3: nseq = (A.qb - 1) / A.bc - A.qa / A.bc + 1; maxq = std::min(A.bc, nq); break;
        case 2: nseq = std::min(A.bc, nq); maxq = (nq + A.bc - 1) / A.bc; break;
        default: break;
    }
    Q.tiles_per_seq = (maxq + 63) / 64;
    if (r.stage_bytes == 4) return r.tile_dh == 160 ? launch_attn_mma<160, false>(A, Q, nseq, n, w, ld, stream)
                                                    : launch_attn_mma<256, false>(A, Q, nseq, n, w, ld, stream);
    switch (r.tile_dh) {
        case 32: return launch_attn_mma<32, true>(A, Q, nseq, n, w, ld, stream);
        case 64: return launch_attn_mma<64, true>(A, Q, nseq, n, w, ld, stream);
        case 128: return launch_attn_mma<128, true>(A, Q, nseq, n, w, ld, stream);
        default: return launch_attn_mma<256, true>(A, Q, nseq, n, w, ld, stream);
    }
}

// dynamic shared memory of the scalar kernels: q and one score per key
size_t scalar_attn_smem(const AttnFwd& A) { return (size_t)(A.dh + fwd_max_keys(A)) * 4; }
constexpr size_t kScalarAttnSmemMax = 64 * 1024;

// One layer's attention, as the prefill runs it: the forward output of positions [A.qa, A.qb) into A.a (when set) and,
// when w is set (head of a window only), the recorded weights w [n][H][P][ld] (zeroed first: entries outside the pattern
// and rows without keys stay 0).  Both take route r.
int layer_attention(const AttnFwd& A, const jk_prefill_attn_route& r, int n, __half* w, int ld, cudaStream_t stream) {
    const size_t smem = scalar_attn_smem(A);
    if (!r.tensor_cores) {
        if (int rc = set_max_smem_once<attn_fwd_kernel>((int)kScalarAttnSmemMax)) return rc;
        if (int rc = set_max_smem_once<attn_record_kernel>((int)kScalarAttnSmemMax)) return rc;
    }
    if (A.a) {
        if (r.tensor_cores) {
            if (int rc = attn_mma(A, r, n, nullptr, 0, stream)) return rc;
        } else {
            attn_fwd_kernel<<<dim3(A.qb - A.qa, A.H, n), kFwdThreads, smem, stream>>>(A);
            JK_CHECK_CUDA(cudaGetLastError());
        }
    }
    if (w) {
        JK_CHECK_CUDA(cudaMemsetAsync(w, 0, (size_t)n * A.H * A.P * ld * sizeof(__half), stream));
        if (r.tensor_cores) {
            if (int rc = attn_mma(A, r, n, w, ld, stream)) return rc;
        } else {
            attn_record_kernel<<<dim3(A.P, A.H, n), kFwdThreads, smem, stream>>>(A, w, ld);
            JK_CHECK_CUDA(cudaGetLastError());
        }
    }
    return 0;
}

// ---- K, V of the given positions -> the caches the decode kernel attends -------------------------------
// Positions [pa, pb) (absolute; qkv row i of a sample is position t0 + i) -> cache row of position p
// (decode_engine.cu attn_geom.wrow); ring layouts keep only the last writer of the range.
__global__ void kv_scatter_kernel(const __half* __restrict__ qkv, __half* __restrict__ kc, __half* __restrict__ vc, int n,
                                  int P, int t0, int pa, int pb, int S, int H, int dh, int dhp, int rows, int attn_func,
                                  int bc, int blocks, int prime) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int np = pb - pa;
    if (i >= (size_t)n * np * S) return;
    const int cs = (int)(i % S);
    const int m = (int)(i / S), b = m / np, p = pa + m % np;
    const int h = cs / dh, d = cs % dh;
    int wrow = -1;
    switch (attn_func) {
        case 0: wrow = p; break;
        case 1: wrow = (p + bc >= pb) ? p % bc : -1; break;
        case 2: wrow = (p % bc) * blocks + p / bc; break;
        case 3: wrow = (p + 2 * bc >= pb) ? ((p / bc) & 1) * bc + p % bc : -1; break;
        case 7: wrow = (p < prime) ? p : -1; break;
    }
    if (wrow < 0) return;
    const size_t dst = (((size_t)b * H + h) * rows + wrow) * dhp + d;
    const __half* src = qkv + ((size_t)b * P + (p - t0)) * 3 * S + cs;
    kc[dst] = src[S];
    vc[dst] = src[2 * S];
}

__global__ void rows_to_float_kernel(const __half* __restrict__ x, float* __restrict__ y, size_t cnt) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < cnt) y[i] = __half2float(x[i]);
}

__global__ void set_position_kernel(int* t, int v) { *t = v; }

// ---- activations of one layer (jk_act_capture, jk_pool_rows_f32): fp32 rows of [t0, t1), or their mean -------------
// One CTA = one sample x a strip of 64 columns; 256 threads = 32 position slots x 8 threads of 8 columns.  Slot s walks
// positions t0 + s, t0 + s + 32, ... and sums in fp64; the 32 slot sums of a column are then added in slot order.  That
// order depends on neither the batch nor the device, so a sample's mean has the same bits alone and in any batch.
constexpr int kActCols = 64, kActSlots = 32;

__device__ __forceinline__ void load8(const __half* p, float (&v)[8], int) {     // the prefill's rows: width % 8 == 0
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = __half2float(h[e]);
}
__device__ __forceinline__ void load8(const float* p, float (&v)[8], int m) {   // any width: m valid columns
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = e < m ? p[e] : 0.f;
}

template <typename T, bool POOL>
__global__ void __launch_bounds__(256) act_rows_kernel(const T* __restrict__ x, int P, int W, int t0, int t1,
                                                       const float* __restrict__ xc, long long xcl, float* __restrict__ out) {
    __shared__ double red[kActSlots][kActCols];
    const int b = blockIdx.y, tid = threadIdx.x, s = tid >> 3, c8 = (tid & 7) * 8;
    const int c = blockIdx.x * kActCols + c8;
    const int m = min(8, W - c);                          // columns of this thread (<= 0: none)
    double acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.0;
    if (m > 0) {
#pragma unroll 4
        for (int t = t0 + s; t < t1; t += kActSlots) {
            float v[8];
            load8(x + ((size_t)b * P + t) * W + c, v, m);
            if (xc) {
                const float* r = xc + ((size_t)b * xcl + (xcl > 1 ? t : 0)) * W + c;
#pragma unroll
                for (int e = 0; e < 8; ++e) if (e < m) v[e] += r[e];
            }
            if (POOL) {
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] += (double)v[e];
            } else {                                      // width % 8 == 0 here (the prefill's rows)
                float4* o = reinterpret_cast<float4*>(out + ((size_t)b * (t1 - t0) + (t - t0)) * W + c);
                o[0] = make_float4(v[0], v[1], v[2], v[3]);
                o[1] = make_float4(v[4], v[5], v[6], v[7]);
            }
        }
    }
    if (!POOL) return;
#pragma unroll
    for (int e = 0; e < 8; ++e) red[s][c8 + e] = acc[e];
    __syncthreads();
    const int col = blockIdx.x * kActCols + tid;
    if (tid < kActCols && col < W) {
        double sum = 0.0;
        for (int k = 0; k < kActSlots; ++k) sum += red[k][tid];
        out[(size_t)b * W + col] = (float)(sum / (double)(t1 - t0));
    }
}

template <typename T>
int launch_act_rows(const T* x, int n, int P, int W, int t0, int t1, const float* xc, long long xcl, int pool, float* out,
                    cudaStream_t stream) {
    const dim3 grid((unsigned)((W + kActCols - 1) / kActCols), (unsigned)n);
    if (pool) act_rows_kernel<T, true><<<grid, 256, 0, stream>>>(x, P, W, t0, t1, xc, xcl, out);
    else act_rows_kernel<T, false><<<grid, 256, 0, stream>>>(x, P, W, t0, t1, xc, xcl, out);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" int jk_pool_rows_f32(const float* x, int n, int P, int width, int t0, int t1, const float* x_cond,
                                int64_t x_cond_len, float* out, jk_stream_t stream) {
    JK_REQUIRE(x && out, "null argument");
    JK_REQUIRE(n >= 1 && P >= 1 && width >= 1, "empty rows (n %d, P %d, width %d)", n, P, width);
    JK_REQUIRE(t0 >= 0 && t0 < t1 && t1 <= P, "positions [%d, %d) empty or outside [0, %d)", t0, t1, P);
    JK_REQUIRE(!x_cond || x_cond_len == 1 || x_cond_len >= t1, "x_cond_len %lld: 1, or at least t1 = %d rows",
               (long long)x_cond_len, t1);
    JK_REQUIRE(((uintptr_t)out & 15) == 0, "out must be 16-byte aligned");
    return launch_act_rows<float>(x, n, P, width, t0, t1, x_cond, x_cond ? x_cond_len : 1, 1, out, (cudaStream_t)stream);
}

extern "C" int jk_prefill_attention_f16(const jk_prefill_attn_args* a, jk_prefill_attn_route* taken, jk_stream_t stream) {
    JK_REQUIRE(a, "null argument");
    const int f = a->attn_func;
    JK_REQUIRE(f == 0 || f == 1 || f == 2 || f == 3 || f == 6 || f == 7, "attn_func %d (0, 1, 2, 3, 6 or 7)", f);
    JK_REQUIRE(a->n >= 1 && a->P >= 1 && a->heads >= 1 && a->dh >= 1, "empty shape (n %d, P %d, heads %d, dh %d)", a->n, a->P,
               a->heads, a->dh);
    JK_REQUIRE(a->dh <= a->dh_pad && a->dh_pad % 16 == 0, "dh_pad %d: a multiple of 16, at least dh %d", a->dh_pad, a->dh);
    JK_REQUIRE(f < 1 || f > 3 || a->bc >= 1, "attn_func %d needs a block length bc >= 1 (got %d)", f, a->bc);
    JK_REQUIRE(f != 7 || a->prime >= 1, "attn_func 7 needs prime >= 1 (got %d)", a->prime);
    JK_REQUIRE(f != 6 || (a->enc_rows >= 1 && a->k_cache && a->v_cache), "attn_func 6 needs enc_rows >= 1 (got %d) and both caches",
               a->enc_rows);
    JK_REQUIRE(!a->w || a->ld >= 1, "recorded weights need ld >= 1 (got %d)", a->ld);
    JK_REQUIRE(a->out || a->w, "neither out nor w: nothing to compute");
    JK_REQUIRE(a->qkv, "null qkv");
    JK_REQUIRE((((uintptr_t)a->qkv | (uintptr_t)a->out | (uintptr_t)a->k_cache | (uintptr_t)a->v_cache) & 15) == 0,
               "qkv, out and the caches must be 16-byte aligned");
    JK_REQUIRE(a->route == 0 || a->route == 1, "route %d (0: the prefill's choice, 1: the scalar kernels)", a->route);
    const int t0 = a->q_offset;
    const bool cont = t0 > 0 || a->cache_rows > 0;          // a continuation: keys from the caches
    JK_REQUIRE(t0 >= 0 && a->cache_rows >= 0, "q_offset %d and cache_rows %d must be >= 0", t0, a->cache_rows);
    if (cont && f != 6) {
        int need = 0;
        switch (f) {
            case 0: need = t0 + a->P; break;
            case 1: need = a->bc; break;
            case 2: need = a->bc * a->blocks; break;
            case 3: need = 2 * a->bc; break;
            case 7: need = a->prime; break;
        }
        JK_REQUIRE(a->k_cache && a->v_cache, "a continuation (q_offset %d, cache_rows %d) reads its keys from both caches",
                   t0, a->cache_rows);
        JK_REQUIRE(f != 2 || (a->blocks >= 1 && t0 + a->P <= a->bc * a->blocks),
                   "attn_func 2 needs blocks >= 1 (got %d) and positions up to bc * blocks = %d (got %d)", a->blocks,
                   a->bc * a->blocks, t0 + a->P);
        JK_REQUIRE(a->cache_rows >= need, "attn_func %d reads %d cache rows at positions [%d, %d), cache_rows is %d", f,
                   need, t0, t0 + a->P, a->cache_rows);
    }
    JK_REQUIRE(!cont || !a->w, "recorded weights are computed at the head of a window only (q_offset 0, cache_rows 0)");
    AttnFwd A;
    A.qkv = (const __half*)a->qkv; A.a = (__half*)a->out; A.kc = (const __half*)a->k_cache; A.vc = (const __half*)a->v_cache;
    A.P = a->P; A.S = a->heads * a->dh; A.H = a->heads; A.dh = a->dh; A.bc = a->bc; A.attn_func = f; A.prime = a->prime;
    A.q_stride = f == 6 ? A.S : 3 * A.S; A.enc_rows = f == 6 ? a->enc_rows : 0; A.dhp = a->dh_pad; A.scale2 = attn_scale2(a->dh);
    A.qoff = t0; A.qa = t0; A.qb = t0 + a->P; A.cache = cont; A.rows = a->cache_rows; A.blocks = a->blocks;
    const jk_prefill_attn_route r = attn_route(A, a->route == 1);
    JK_REQUIRE(r.tensor_cores || scalar_attn_smem(A) <= kScalarAttnSmemMax,
               "the scalar kernels hold dh + the keys of a query = %d floats in shared memory (at most %d)",
               a->dh + fwd_max_keys(A), (int)(kScalarAttnSmemMax / 4));
    if (int rc = layer_attention(A, r, a->n, (__half*)a->w, a->ld, (cudaStream_t)stream)) return rc;
    if (taken) *taken = r;
    return 0;
}

extern "C" int jk_prior_prefill_capacity(const jk_prior* p, int* max_positions) {
    JK_REQUIRE(p && max_positions, "null argument");
    *max_positions = p->pf_len;
    return 0;
}

extern "C" int jk_prior_prefill(jk_prior* p, const jk_prefill_args* a, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(p && a, "null argument");
    const jk_prior_config& c = p->cfg;
    const EngineDev& E = p->host;
    JK_REQUIRE(p->pf_len > 0, "this configuration has no chunked prefill (needs width, n_state, mlp_width >= 64 and %% 8 == 0): "
                              "step the given tokens through jk_prior_step");
    JK_REQUIRE(p->t_host >= 0, "the last prefill stopped early (n_layers) and left later layers' caches unfilled: "
                               "call jk_prior_reset first");
    const int t0 = p->t_host;      // > 0: a continuation of the rows' K / V caches
    const int n = a->n_samples, P = a->n_positions;
    JK_REQUIRE(n >= 1 && n <= c.max_batch, "n_samples %d out of range (max_batch %d)", n, c.max_batch);
    JK_REQUIRE(P >= 1 && P <= p->pf_len, "n_positions %d out of range (capacity %d)", P, p->pf_len);
    JK_REQUIRE(t0 + P <= c.n_ctx, "positions [%d, %d) run past the context (n_ctx %d)", t0, t0 + P, c.n_ctx);
    JK_REQUIRE((P == 1 && t0 == 0) || a->tokens, "tokens required");
    JK_REQUIRE(t0 == 0 || (a->n_record == 0 && a->n_capture == 0 && (a->n_layers == 0 || a->n_layers == c.depth)),
               "record, capture and n_layers < depth are head-of-window features (the engine is at %d, not 0)", t0);
    JK_REQUIRE(E.pos_emb && E.x_emb, "embeddings not set (jk_prior_set_embeddings)");
    JK_REQUIRE(a->x_cond_len == 0 || a->x_cond_len == 1 || a->x_cond_len == c.n_ctx, "x_cond_len must be 1 or n_ctx");
    const int W = c.width, S = c.n_state, Mw = c.mlp_width, H = c.heads;
    const int rows = n * P;
    JK_REQUIRE(a->n_layers >= 0 && a->n_layers <= c.depth, "n_layers %d out of range (0 = all, else 1 .. depth %d)",
               a->n_layers, c.depth);
    const int depth = a->n_layers ? a->n_layers : c.depth;      // layers this call runs
    JK_REQUIRE(a->n_record >= 0 && (a->n_record == 0 || a->record), "record: %d layers but no table", a->n_record);
    const jk_attn_record* rec[JK_MAX_DEPTH] = {};     // per layer: its entry of a->record, or NULL
    for (int i = 0; i < a->n_record; ++i) {
        const jk_attn_record& r = a->record[i];
        JK_REQUIRE(r.layer >= 0 && r.layer < depth, "record: layer %d out of range (depth %d)", r.layer, depth);
        JK_REQUIRE(!rec[r.layer], "record: layer %d listed twice", r.layer);
        JK_REQUIRE(r.ld >= 1, "record: layer %d has ld %d (>= 1 keys per row)", r.layer, r.ld);
        JK_REQUIRE(r.w, "record: layer %d has no output buffer", r.layer);
        rec[r.layer] = &r;
    }
    JK_REQUIRE(a->n_capture >= 0 && (a->n_capture == 0 || a->capture), "capture: %d layers but no table", a->n_capture);
    const jk_act_capture* cap[JK_MAX_DEPTH] = {};     // per layer: its entry of a->capture, or NULL
    for (int i = 0; i < a->n_capture; ++i) {
        const jk_act_capture& k = a->capture[i];
        JK_REQUIRE(k.layer >= 0 && k.layer < depth, "capture: layer %d out of range (%d layers run)", k.layer, depth);
        JK_REQUIRE(!cap[k.layer], "capture: layer %d listed twice", k.layer);
        JK_REQUIRE(k.t0 >= 0 && k.t0 < k.t1 && k.t1 <= P, "capture: layer %d positions [%d, %d) empty or outside [0, %d)",
                   k.layer, k.t0, k.t1, P);
        JK_REQUIRE(k.pool == 0 || k.pool == 1, "capture: layer %d has pool %d (0 or 1)", k.layer, k.pool);
        JK_REQUIRE(k.out, "capture: layer %d has no output buffer", k.layer);
        JK_REQUIRE(((uintptr_t)k.out & 15) == 0, "capture: layer %d output is not 16-byte aligned", k.layer);
        JK_REQUIRE(!k.add_x_cond || a->x_cond, "capture: layer %d adds x_cond, but the call has none", k.layer);
        cap[k.layer] = &k;
    }
    {
        const size_t cnt = (size_t)rows * W;
        embed_rows_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, stream>>>(
            p->pf_x, (const long long*)a->tokens, a->tok_stride, a->y_cond, a->x_cond, a->x_cond_len ? a->x_cond_len : 1,
            E.x_emb, E.pos_emb, E.start_token, n, P, t0, W);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    const unsigned ln_grid = (unsigned)((rows + 7) / 8);
    JK_REQUIRE((size_t)(E.dh + std::max(t0 + P, E.enc_dims)) * 4 <= kScalarAttnSmemMax, "prefill attention tile too large");
    for (int l = 0; l < depth; ++l) {
        const LayerDev& LD = E.layer[l];
        ln_rows_kernel<<<ln_grid, 256, 0, stream>>>(p->pf_x, LD.ln0_g, LD.ln0_b, p->pf_xn, rows, W);
        JK_CHECK_CUDA(cudaGetLastError());
        const bool enc = LD.attn_func == 6;       // c_attn gives q only; K / V are the encoder's (already in the cache)
        const int q_stride = enc ? S : 3 * S;
        int rc = gemm_f16_tc(p->pf_xn, p->wt[0][l], LD.b_qkv, nullptr, p->pf_qkv, rows, q_stride, W, 0, stream);
        if (rc) return rc;
        AttnFwd A;
        A.qkv = p->pf_qkv; A.a = p->pf_a; A.P = P; A.S = S; A.H = H; A.dh = E.dh; A.bc = E.bc; A.attn_func = LD.attn_func;
        A.prime = E.prime_pad; A.scale2 = E.scale2; A.q_stride = q_stride; A.kc = LD.kc; A.vc = LD.vc; A.enc_rows = E.enc_dims;
        A.dhp = E.dh_pad;
        A.qoff = t0; A.qa = t0; A.qb = t0 + P; A.cache = t0 > 0; A.rows = LD.rows; A.blocks = E.blocks;
        // tensor cores when the head geometry allows (dh even, dh <= 256)
        const jk_prefill_attn_route route = attn_route(A, false);
        auto scatter = [&](int pa, int pb) -> int {
            const size_t cnt = (size_t)n * (pb - pa) * S;
            kv_scatter_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, stream>>>(p->pf_qkv, LD.kc, LD.vc, n, P, t0, pa, pb, S, H,
                                                                                  E.dh, E.dh_pad, LD.rows, LD.attn_func, E.bc,
                                                                                  E.blocks, E.prime_pad);
            JK_CHECK_CUDA(cudaGetLastError());
            return 0;
        };
        if (t0 == 0) {
            // queries and keys from pf_qkv; the recorded weights read q / K only, so they are taken here, before the next
            // layer overwrites pf_qkv
            const jk_attn_record* r = rec[l];
            rc = layer_attention(A, route, n, r ? (__half*)r->w : nullptr, r ? r->ld : 0, stream);
            if (rc) return rc;
            if (!enc && (rc = scatter(0, P))) return rc;
        } else if (LD.attn_func == 1 || LD.attn_func == 3) {
            // ring layouts: a block's rows overwrite rows earlier blocks' queries read, so the chunk goes block by block,
            // each block's K / V into the cache and then its queries over the cache
            for (int pa = t0; pa < t0 + P; pa = (pa / E.bc + 1) * E.bc) {
                const int pb = std::min(t0 + P, (pa / E.bc + 1) * E.bc);
                if ((rc = scatter(pa, pb))) return rc;
                A.qa = pa; A.qb = pb;
                if ((rc = layer_attention(A, route, n, nullptr, 0, stream))) return rc;
            }
        } else {
            // every position has its own row (0, 2, 7; 6 reads the encoder rows): the whole chunk into the cache first
            if (!enc && (rc = scatter(t0, t0 + P))) return rc;
            if ((rc = layer_attention(A, route, n, nullptr, 0, stream))) return rc;
        }
        rc = gemm_f16_tc(p->pf_a, p->wt[1][l], LD.b_o, p->pf_x, p->pf_x1, rows, W, S, 2, stream);
        if (rc) return rc;
        ln_rows_kernel<<<ln_grid, 256, 0, stream>>>(p->pf_x1, LD.ln1_g, LD.ln1_b, p->pf_xn, rows, W);
        JK_CHECK_CUDA(cudaGetLastError());
        rc = gemm_f16_tc(p->pf_xn, p->wt[2][l], LD.b_1, nullptr, p->pf_g, rows, Mw, W, 1, stream);
        if (rc) return rc;
        rc = gemm_f16_tc(p->pf_g, p->wt[3][l], LD.b_2, p->pf_x1, p->pf_x, rows, W, Mw, 2, stream);
        if (rc) return rc;
        if (const jk_act_capture* k = cap[l]) {         // the layer's output, before the next layer overwrites pf_x
            rc = launch_act_rows<__half>(p->pf_x, n, P, W, k->t0, k->t1, k->add_x_cond ? a->x_cond : nullptr,
                                         a->x_cond_len ? a->x_cond_len : 1, k->pool, k->out, stream);
            if (rc) return rc;
        }
    }
    if (a->h_out) {
        const size_t cnt = (size_t)rows * W;
        rows_to_float_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, stream>>>(p->pf_x, a->h_out, cnt);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    if (depth < c.depth) {      // later layers' caches are not filled: not steppable until jk_prior_reset
        p->t_host = -1;
        return 0;
    }
    set_position_kernel<<<1, 1, 0, stream>>>(E.t, t0 + P);
    JK_CHECK_CUDA(cudaGetLastError());
    p->t_host = t0 + P;
    return 0;
}
