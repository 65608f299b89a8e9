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

// The draw of one row (one CTA): tokens[row * tok_stride + position] and, when s_tok is given, *s_tok (visible to the
// whole CTA after a __syncthreads).  max_per: bins each thread owns (compile-time bound keeps e[] in registers)
template <int MAX_PER>
__device__ __forceinline__ void draw_row(const float* __restrict__ logits, long long lstride, int bins, float temp,
                                         unsigned long long seed, int position, long long* __restrict__ tokens,
                                         long long tok_stride, int* s_tok) {
    __shared__ float s_red[kThreads / 32];
    __shared__ float s_scan[kThreads / 32];
    __shared__ float s_bcast[2];
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* l = logits + (long long)row * lstride;
    const int per = (bins + kThreads - 1) / kThreads;
    const int b0 = tid * per;
    // x / temp as torch computes it on a GPU for a scalar divisor: x * (1 / temp) (BinaryDivTrueKernel: a * reciprocal(b))
    const float inv_temp = 1.0f / temp;
    float e[MAX_PER];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < MAX_PER; ++j) {
        const int b = b0 + j;
        e[j] = (j < per && b < bins) ? __ldcg(l + b) * inv_temp : -INFINITY;
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
    draw_row<MAX_PER>(logits, lstride, bins, temp, seed, position, tokens, tok_stride, nullptr);
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
    __shared__ float s_red[kThreads / 32];
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (logits) draw_row<MAX_PER>(logits, lstride, bins, temp, seed, position, tokens, tok_stride, &s_tok);
    else if (tid == 0) s_tok = (int)tokens[(long long)row * tok_stride + position];
    const float* r = raw + (long long)row * rstride;
    float mx = -INFINITY;
    for (int b = tid; b < bins; b += kThreads) mx = fmaxf(mx, __ldcg(r + b));
    mx = jk::warp_max(mx);
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();                                   // also publishes s_tok
    mx = s_red[0];
#pragma unroll
    for (int w = 1; w < kThreads / 32; ++w) mx = fmaxf(mx, s_red[w]);
    float se = 0.f;
    for (int b = tid; b < bins; b += kThreads) se += expf(__ldcg(r + b) - mx);
    se = jk::warp_sum(se);
    __syncthreads();                                   // every thread has read the maxima
    if (lane == 0) s_red[warp] = se;
    __syncthreads();
    if (tid == 0) {
        float total = 0.f;
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) total += s_red[w];
        const int tok = s_tok;               // a given token outside [0, bins) has no likelihood: nan
        logp[(long long)row * logp_stride + position] =
            (tok >= 0 && tok < bins) ? __ldcg(r + tok) - mx - logf(total) : __int_as_float(0x7fffffff);
    }
}


// ---- top-k / nucleus filtering (reference transformer/ops.py:113-142) -----------------------------------
// out = logits / temp with every entry outside the kept set replaced by -inf.  One CTA per row: the row is sorted
// (descending, bitonic, shared memory) and the kept set is "values >= cutoff":
//   top_k : cutoff = k-th largest value (ops.py:125-128: logits < topk(logits, k)[..., -1:] are removed)
//   top_p : sorted index j is removed iff the softmax mass of sorted[0 .. j-1] exceeds top_p (ops.py:130-140: the
//           removal mask is shifted right by one, the largest entry always stays); cutoff = last kept value
constexpr int kFilterMax = 4096;

__global__ void __launch_bounds__(kThreads)
filter_logits_kernel(const float* __restrict__ logits, long long lstride, int bins, float temp, int top_k, float top_p,
                     float* __restrict__ out, long long ostride) {
    __shared__ float s[kFilterMax];
    __shared__ float s_scan[kThreads / 32];
    __shared__ int s_keep;
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* l = logits + (long long)row * lstride;
    int P = 1;
    while (P < bins) P <<= 1;
    const float inv_temp = 1.0f / temp;         // torch's x / scalar on a GPU: x * (1 / scalar)
    for (int i = tid; i < P; i += kThreads) s[i] = (i < bins) ? __ldcg(l + i) * inv_temp : -INFINITY;
    __syncthreads();
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
    float cutoff;
    if (top_k > 0) {
        cutoff = s[min(top_k, bins) - 1];
    } else {
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
        cutoff = s[s_keep - 1];
    }
    float* o = out + (long long)row * ostride;
    for (int i = tid; i < bins; i += kThreads) {
        const float v = __ldcg(l + i) * inv_temp;
        o[i] = (v < cutoff) ? -INFINITY : v;
    }
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
