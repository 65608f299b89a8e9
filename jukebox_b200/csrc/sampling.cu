// Token sampling for the autoregressive loop: x / temp -> Categorical(logits=x).sample()
// (reference jukebox/prior/autoregressive.py:233-235 and :343-345) as ONE launch per position instead
// of the ~10 elementwise/reduction launches the torch expression costs between two decode steps.
//
// One CTA per sample row.  Each thread owns a contiguous run of bins so that the inclusive scan of
// exp(v - max) is the CDF in bin order; the token is the first bin whose CDF reaches u * total,
// u in (0, 1] from Philox4x32-10 keyed by (seed) and countered by (position, row) - the draw for a
// given (seed, position, row) does not depend on launch order or on the other rows.
#include "common.cuh"
#include "../../include/jkb200.h"

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ uint32_t philox_u32(uint64_t seed, uint32_t c0, uint32_t c1) {
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    uint32_t c[4] = {c0, c1, 0x6a6b3230u, 0u};
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
        const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c[0];
}

// One row's entry b: from global memory through L2 (read once, not kept in L1), or from shared memory
template <bool kGlobal>
__device__ __forceinline__ float load_row(const float* __restrict__ l, int b) {
    if constexpr (kGlobal) return __ldcg(l + b);
    else return l[b];
}

// The draw of one row (one CTA) from its logits l[0 .. bins) (global memory, or shared memory with kGlobal = false):
// tokens[row * tok_stride + position] and, when s_tok is given, *s_tok (visible to the whole CTA after a
// __syncthreads).  row keys the Philox counter.  max_per: bins each thread owns (compile-time bound keeps e[] in
// registers)
template <int MAX_PER, bool kGlobal = true>
__device__ __forceinline__ void draw_row(const float* __restrict__ l, int row, int bins, float temp,
                                         unsigned long long seed, int position, long long* __restrict__ tokens,
                                         long long tok_stride, int* s_tok) {
    __shared__ float s_red[kThreads / 32];
    __shared__ float s_scan[kThreads / 32];
    __shared__ float s_bcast[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per = (bins + kThreads - 1) / kThreads;
    const int b0 = tid * per;
    // x / temp as torch computes it on a GPU for a scalar divisor: x * (1 / temp) (BinaryDivTrueKernel: a * reciprocal(b))
    const float inv_temp = 1.0f / temp;
    float e[MAX_PER];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < MAX_PER; ++j) {
        const int b = b0 + j;
        e[j] = (j < per && b < bins) ? load_row<kGlobal>(l, b) * inv_temp : -INFINITY;
        mx = fmaxf(mx, e[j]);
    }
    mx = jk::warp_max(mx);
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();
    mx = s_red[0];
#pragma unroll
    for (int w = 1; w < kThreads / 32; ++w) mx = fmaxf(mx, s_red[w]);
    float local = 0.f;
#pragma unroll
    for (int j = 0; j < MAX_PER; ++j) {
        e[j] = (e[j] == -INFINITY) ? 0.f : __expf(e[j] - mx);
        local += e[j];
    }
    // inclusive scan of the per-thread sums: warp shuffle scan, then the warp totals
    float incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_scan[warp] = incl;
    __syncthreads();
    float woff = 0.f, total = 0.f;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
        if (w < warp) woff += s_scan[w];
        total += s_scan[w];
    }
    incl += woff;
    const float excl = incl - local;
    if (tid == 0) {
        const uint32_t r = philox_u32(seed, (uint32_t)position, (uint32_t)row);
        s_bcast[0] = (float)((r >> 8) + 1u) * (1.0f / 16777216.0f) * total;    // u in (2^-24, 1]
    }
    if (tid == 0) s_bcast[1] = __int_as_float(0x7fffffff);
    __syncthreads();
    const float target = s_bcast[0];
    // the owning thread: first whose inclusive sum reaches the target (ties between threads with an
    // empty run cannot win: local > 0 is required)
    const bool mine = local > 0.f && excl < target && incl >= target;
    const bool last_resort = (tid == kThreads - 1);
    int pick = -1;
    if (mine) {
        float run = excl;
        int fallback = -1;
#pragma unroll
        for (int j = 0; j < MAX_PER; ++j) {
            if (e[j] > 0.f) {
                run += e[j];
                fallback = b0 + j;
                if (pick < 0 && run >= target) pick = b0 + j;
            }
        }
        if (pick < 0) pick = fallback;
        tokens[(long long)row * tok_stride + position] = pick;
        if (s_tok) *s_tok = pick;
        s_bcast[1] = 0.f;
    }
    __syncthreads();
    // rounding of woff/incl can leave no owner in a pathological row: take the last bin with mass
    if (s_bcast[1] != 0.f) {
        __shared__ int s_last;
        if (tid == 0) s_last = -1;
        __syncthreads();
        int lastb = -1;
#pragma unroll
        for (int j = 0; j < MAX_PER; ++j)
            if (e[j] > 0.f) lastb = b0 + j;
        if (lastb >= 0) atomicMax(&s_last, lastb);
        __syncthreads();
        if (last_resort) {
            tokens[(long long)row * tok_stride + position] = s_last < 0 ? 0 : s_last;
            if (s_tok) *s_tok = s_last < 0 ? 0 : s_last;
        }
    }
}

template <int MAX_PER>
__global__ void __launch_bounds__(kThreads)
sample_categorical_kernel(const float* __restrict__ logits, long long lstride, int bins, float temp,
                          unsigned long long seed, int position, long long* __restrict__ tokens,
                          long long tok_stride) {
    const int row = blockIdx.x;
    draw_row<MAX_PER>(logits + (long long)row * lstride, row, bins, temp, seed, position, tokens, tok_stride, nullptr);
}

// *out = log_softmax(r[0 .. bins))[*s_tok]: the likelihood at temperature 1 of the unfiltered logits r (global memory, or
// shared memory with kGlobal = false); nan for a token outside [0, bins).  s_tok is read after this function's first
// __syncthreads, so the caller may set it just before the call.
template <bool kGlobal>
__device__ __forceinline__ void store_logp(const float* __restrict__ r, int bins, const int* s_tok, float* out) {
    __shared__ float s_red[kThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float mx = -INFINITY;
    for (int b = tid; b < bins; b += kThreads) mx = fmaxf(mx, load_row<kGlobal>(r, b));
    mx = jk::warp_max(mx);
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();                                   // also publishes *s_tok
    mx = s_red[0];
#pragma unroll
    for (int w = 1; w < kThreads / 32; ++w) mx = fmaxf(mx, s_red[w]);
    float se = 0.f;
    for (int b = tid; b < bins; b += kThreads) se += expf(load_row<kGlobal>(r, b) - mx);
    se = jk::warp_sum(se);
    __syncthreads();                                   // every thread has read the maxima
    if (lane == 0) s_red[warp] = se;
    __syncthreads();
    if (tid == 0) {
        float total = 0.f;
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) total += s_red[w];
        const int tok = *s_tok;
        *out = (tok >= 0 && tok < bins) ? load_row<kGlobal>(r, tok) - mx - logf(total) : __int_as_float(0x7fffffff);
    }
}

// The same draw (logits != NULL) or the given tokens[row, position] (logits == NULL), then
// logp[row, position] = log_softmax(raw[row, :])[token]: the likelihood at temperature 1 of the unfiltered logits
template <int MAX_PER>
__global__ void __launch_bounds__(kThreads)
sample_categorical_scored_kernel(const float* __restrict__ logits, long long lstride, const float* __restrict__ raw,
                                 long long rstride, int bins, float temp, unsigned long long seed, int position,
                                 long long* __restrict__ tokens, long long tok_stride, float* __restrict__ logp,
                                 long long logp_stride) {
    __shared__ int s_tok;
    const int row = blockIdx.x;
    if (logits) draw_row<MAX_PER>(logits + (long long)row * lstride, row, bins, temp, seed, position, tokens, tok_stride,
                                  &s_tok);
    else if (threadIdx.x == 0) s_tok = (int)tokens[(long long)row * tok_stride + position];
    // a given token outside [0, bins) has no likelihood: nan
    store_logp<true>(raw + (long long)row * rstride, bins, &s_tok, logp + (long long)row * logp_stride + position);
}


// ---- top-k / nucleus filtering (reference transformer/ops.py:113-142) -----------------------------------
// out = logits / temp with every entry outside the kept set replaced by -inf.  One CTA per row: the row is sorted
// (descending, bitonic, shared memory) and the kept set is "values >= cutoff":
//   top_k : cutoff = k-th largest value (ops.py:125-128: logits < topk(logits, k)[..., -1:] are removed)
//   top_p : sorted index j is removed iff the softmax mass of sorted[0 .. j-1] exceeds top_p (ops.py:130-140: the
//           removal mask is shifted right by one, the largest entry always stays); cutoff = last kept value
constexpr int kFilterMax = 4096;

// The cutoff of one row (one CTA): s[0 .. P) holds the row / temp, padded with -inf from bins to P (P the power of two
// >= bins), visible to the whole CTA.  s is sorted in place (descending) and the cutoff returned to every thread; the
// kept set is "value >= cutoff".  top_k > 0 or top_p > 0, not both.
__device__ __forceinline__ float filter_cutoff(float* s, int P, int bins, int top_k, float top_p) {
    __shared__ float s_scan[kThreads / 32];
    __shared__ int s_keep;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P; i += kThreads) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const float a = s[i], b = s[ixj];
                    const bool desc = ((i & k) == 0);
                    if (desc ? (a < b) : (a > b)) { s[i] = b; s[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
    if (top_k > 0) return s[min(top_k, bins) - 1];
    // exclusive softmax mass in front of each sorted entry; each thread owns a contiguous run
    const int per = P / kThreads > 0 ? P / kThreads : 1;
    const int b0 = tid * per;
    const float mx = s[0];
    float local = 0.f;
    for (int j = 0; j < per; ++j) {
        const int i = b0 + j;
        if (i < P) local += (s[i] == -INFINITY) ? 0.f : __expf(s[i] - mx);
    }
    float incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_scan[warp] = incl;
    if (tid == 0) s_keep = 1;
    __syncthreads();
    float woff = 0.f, total = 0.f;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
        if (w < warp) woff += s_scan[w];
        total += s_scan[w];
    }
    float run = incl + woff - local;                       // mass strictly before b0
    int keep = 0;                                          // entries of this run that stay
    for (int j = 0; j < per; ++j) {
        const int i = b0 + j;
        if (i < bins) {
            if (i == 0 || !(run / total > top_p)) keep = i + 1;
            run += (s[i] == -INFINITY) ? 0.f : __expf(s[i] - mx);
        }
    }
    // the kept set is a prefix (mass is monotone): its length is the largest keep over the threads
    if (keep > 0) atomicMax(&s_keep, keep);
    __syncthreads();
    return s[s_keep - 1];
}

__global__ void __launch_bounds__(kThreads)
filter_logits_kernel(const float* __restrict__ logits, long long lstride, int bins, float temp, int top_k, float top_p,
                     float* __restrict__ out, long long ostride) {
    __shared__ float s[kFilterMax];
    const int row = blockIdx.x, tid = threadIdx.x;
    const float* l = logits + (long long)row * lstride;
    int P = 1;
    while (P < bins) P <<= 1;
    const float inv_temp = 1.0f / temp;         // torch's x / scalar on a GPU: x * (1 / scalar)
    for (int i = tid; i < P; i += kThreads) s[i] = (i < bins) ? __ldcg(l + i) * inv_temp : -INFINITY;
    __syncthreads();
    const float cutoff = filter_cutoff(s, P, bins, top_k, top_p);
    float* o = out + (long long)row * ostride;
    for (int i = tid; i < bins; i += kThreads) {
        const float v = __ldcg(l + i) * inv_temp;
        o[i] = (v < cutoff) ? -INFINITY : v;
    }
}

// ---- guided draw: one token from two conditionings ----------------------------------------------------------------
// Pair r (one CTA): g = c[r] + s (c[r] - u[r]) in fp32, each operation rounded on its own (no FMA contraction), so that
// torch's `c + s * (c - u)` gives the same bits; then exactly jk_filter_logits(g, temp, top_k, top_p) (when a filter is
// set) and jk_sample_categorical's draw of row r, the token written to tokens[r] and tokens_alt[r].  Every operand row
// is read from global memory once: c and u into g, c (as the scored row) into s_raw when logp is given.
// Dynamic shared memory: g [bins], the sort buffer [P] with a filter, the raw row [bins] with logp.
template <int MAX_PER>
__global__ void __launch_bounds__(kThreads)
sample_guided_kernel(const float* __restrict__ c, long long c_stride, const float* __restrict__ u, long long u_stride,
                     int bins, float s, float temp, int top_k, float top_p, unsigned long long seed, int position,
                     long long* __restrict__ tokens, long long tok_stride, long long* __restrict__ tokens_alt,
                     long long tok_alt_stride, const float* __restrict__ raw, float* __restrict__ logp,
                     long long logp_stride) {
    extern __shared__ float s_dyn[];
    __shared__ int s_tok;
    const int row = blockIdx.x, tid = threadIdx.x;
    const bool filter = top_k > 0 || top_p > 0.f;
    int P = 1;
    while (P < bins) P <<= 1;
    float* s_g = s_dyn;
    float* s_sort = s_g + bins;
    float* s_raw = s_sort + (filter ? P : 0);
    const float* cr = c + (long long)row * c_stride;
    const float* ur = u + (long long)row * u_stride;
    const float* rr = logp ? raw + (long long)row * c_stride : nullptr;
    const float inv_temp = 1.0f / temp;
    for (int i = tid; i < bins; i += kThreads) {
        const float cv = __ldcg(cr + i);
        const float g = __fadd_rn(cv, __fmul_rn(s, __fsub_rn(cv, __ldcg(ur + i))));
        s_g[i] = g;
        if (filter) s_sort[i] = g * inv_temp;
        if (rr) s_raw[i] = (rr == cr) ? cv : __ldcg(rr + i);
    }
    if (filter)
        for (int i = bins + tid; i < P; i += kThreads) s_sort[i] = -INFINITY;
    __syncthreads();
    float draw_temp = temp;
    if (filter) {   // jk_filter_logits' output, then the draw at temperature 1 as the sampling loop runs it
        const float cutoff = filter_cutoff(s_sort, P, bins, top_k, top_p);
        for (int i = tid; i < bins; i += kThreads) {
            const float v = s_g[i] * inv_temp;
            s_g[i] = (v < cutoff) ? -INFINITY : v;
        }
        __syncthreads();
        draw_temp = 1.0f;
    }
    draw_row<MAX_PER, false>(s_g, row, bins, draw_temp, seed, position, tokens, tok_stride, &s_tok);
    __syncthreads();
    if (tid == 0) tokens_alt[(long long)row * tok_alt_stride + position] = s_tok;
    if (logp) store_logp<false>(s_raw, bins, &s_tok, logp + (long long)row * logp_stride + position);
}

}  // namespace

extern "C" int jk_sample_categorical(const float* logits, int64_t logits_stride, int n, int bins, float temp,
                                     uint64_t seed, int position, int64_t* tokens, int64_t tok_stride,
                                     jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(logits && tokens, "null argument");
    JK_REQUIRE(bins >= 1 && bins <= 32 * kThreads, "bins must be in [1, %d]", 32 * kThreads);
    JK_REQUIRE(temp > 0.f, "temp must be positive");
    JK_REQUIRE(position >= 0, "negative position");
    if (n == 0) return 0;
    const int per = (bins + kThreads - 1) / kThreads;
#define JK_LAUNCH(MP)                                                                              \
    sample_categorical_kernel<MP><<<n, kThreads, 0, stream>>>(logits, (long long)logits_stride, bins, temp, \
                                                              (unsigned long long)seed, position,  \
                                                              (long long*)tokens, (long long)tok_stride)
    if (per <= 4) JK_LAUNCH(4);
    else if (per <= 8) JK_LAUNCH(8);
    else if (per <= 16) JK_LAUNCH(16);
    else JK_LAUNCH(32);
#undef JK_LAUNCH
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_sample_categorical_scored(const float* logits, int64_t logits_stride, const float* raw,
                                            int64_t raw_stride, int n, int bins, float temp, uint64_t seed, int position,
                                            int64_t* tokens, int64_t tok_stride, float* logp, int64_t logp_stride,
                                            jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(raw && tokens && logp, "null argument");
    JK_REQUIRE(bins >= 1 && bins <= 32 * kThreads, "bins must be in [1, %d]", 32 * kThreads);
    JK_REQUIRE(temp > 0.f, "temp must be positive");
    JK_REQUIRE(position >= 0, "negative position");
    if (n == 0) return 0;
    const int per = (bins + kThreads - 1) / kThreads;
#define JK_LAUNCH(MP)                                                                                                \
    sample_categorical_scored_kernel<MP><<<n, kThreads, 0, stream>>>(                                                \
        logits, (long long)logits_stride, raw, (long long)raw_stride, bins, temp, (unsigned long long)seed, position, \
        (long long*)tokens, (long long)tok_stride, logp, (long long)logp_stride)
    if (per <= 4) JK_LAUNCH(4);
    else if (per <= 8) JK_LAUNCH(8);
    else if (per <= 16) JK_LAUNCH(16);
    else JK_LAUNCH(32);
#undef JK_LAUNCH
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_filter_logits(const float* logits, int64_t logits_stride, int n, int bins, float temp, int top_k,
                                float top_p, float* out, int64_t out_stride, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(logits && out, "null argument");
    JK_REQUIRE(bins >= 1 && bins <= kFilterMax, "bins must be in [1, %d]", kFilterMax);
    JK_REQUIRE(temp > 0.f, "temp must be positive");
    JK_REQUIRE(top_k >= 0 && top_p >= 0.f && top_p <= 1.f, "top_k >= 0 and 0 <= top_p <= 1 expected");
    JK_REQUIRE((top_k == 0) != (top_p == 0.f), "exactly one of top_k / top_p must be set (ops.py:122)");
    if (n == 0) return 0;
    filter_logits_kernel<<<n, kThreads, 0, stream>>>(logits, (long long)logits_stride, bins, temp, top_k, top_p, out,
                                                     (long long)out_stride);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_sample_guided(const float* c, int64_t c_stride, const float* u, int64_t u_stride, int n, int bins,
                                float s, float temp, int top_k, float top_p, uint64_t seed, int position, int64_t* tokens,
                                int64_t tok_stride, int64_t* tokens_alt, int64_t tok_alt_stride, const float* raw,
                                float* logp, int64_t logp_stride, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(c && u && tokens && tokens_alt, "null argument");
    JK_REQUIRE((raw == nullptr) == (logp == nullptr), "raw and logp are both given or both NULL");
    JK_REQUIRE(n >= 0, "negative pair count %d", n);
    JK_REQUIRE(bins >= 1 && bins <= kFilterMax, "bins must be in [1, %d]", kFilterMax);
    JK_REQUIRE(temp > 0.f, "temp must be positive");
    JK_REQUIRE(isfinite(s), "guidance weight s must be finite");
    JK_REQUIRE(top_k >= 0 && top_p >= 0.f && top_p <= 1.f, "top_k >= 0 and 0 <= top_p <= 1 expected");
    JK_REQUIRE(top_k == 0 || top_p == 0.f, "at most one of top_k / top_p may be set (ops.py:122)");
    JK_REQUIRE(position >= 0, "negative position");
    if (n == 0) return 0;
    const bool filter = top_k > 0 || top_p > 0.f;
    int P = 1;
    while (P < bins) P <<= 1;
    const size_t smem = sizeof(float) * ((size_t)bins + (filter ? P : 0) + (logp ? bins : 0));
    const int per = (bins + kThreads - 1) / kThreads;
#define JK_LAUNCH(MP)                                                                                               \
    do {                                                                                                            \
        if (smem > 40 * 1024)                                                                                       \
            JK_CHECK_CUDA(cudaFuncSetAttribute(sample_guided_kernel<MP>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                               (int)(3 * kFilterMax * sizeof(float))));                              \
        sample_guided_kernel<MP><<<n, kThreads, smem, stream>>>(                                                    \
            c, (long long)c_stride, u, (long long)u_stride, bins, s, temp, top_k, top_p, (unsigned long long)seed,  \
            position, (long long*)tokens, (long long)tok_stride, (long long*)tokens_alt, (long long)tok_alt_stride,  \
            raw, logp, (long long)logp_stride);                                                                     \
    } while (0)
    if (per <= 4) JK_LAUNCH(4);
    else if (per <= 8) JK_LAUNCH(8);
    else JK_LAUNCH(16);
#undef JK_LAUNCH
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}
