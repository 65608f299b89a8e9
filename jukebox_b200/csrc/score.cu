// Log-probabilities of given tokens straight from the activations:
//
//   logp[m] = z[m, target[m]] - log sum_b exp(z[m, b]),   z = h . x_out^T  (prior/autoregressive.py: x_out, no bias)
//
// without the [M, bins] logits ever reaching HBM.  The head kernel runs conv_wide_kernel's streamed-weight pipeline
// (streamed_pipeline, split_tma.cuh) with its own loads and epilogue (HeadJob): hi.w_hi + hi.w_lo + lo.w_hi of fp16
// halves (22 significant bits per operand), x_out scaled by 2^8 before its split so that the weight remainders stay
// normal, warpgroup MMAs with fp32 accumulation, and every 64-wide K block's partial promoted into an fp32 register sum
// with ordinary adds (the tensor core's own accumulation alone drifts to ~2e-5 of the output scale over long K).
//
// Work items are (128 rows x 128 bins) tiles, numbered row-tile major so that the CTAs working on the bin tiles of one
// row tile at the same time share its activation rows in L2.  One persistent CTA per SM, four roles over mbarriers:
//   warp 12        TMA producer: per K block the fp32 activations [128 x 64] and the hi / lo planes of the weight
//                  block [128 x 64] (128-byte swizzle) into a 3-stage ring;
//   warps 8-11     converters: fp32 block -> hi / lo fp16 planes in place; any value the fp16 split cannot hold
//                  (|h| > 65504, inf, nan) raises the status word instead of saturating;
//   warps 0-7      consumers, rows 0-63 / 64-127: 12 wgmma m64n128k16 per K block into a zeroed partial, added to the
//                  tile's fp32 sum.  The epilogue reduces each row of the tile to (max, sum exp(z - max)) over the bins
//                  it covers - one pair per (row, bin tile) in the workspace - and stores z[m, target] from the one
//                  tile that holds the target.
// A second kernel combines the pairs of a row in bin-tile order: the result does not depend on the other rows, the
// grid or the schedule, so a row gives the same bits alone and in any batch.
//
// jk_xout_stats runs the same mainloop (xout_head_kernel<true>) with a wider epilogue: beside the pair it stores
// u = sum (z - max) exp(z - max) and the tile's K largest (z, bin), and its combine adds the entropy (fp64) and the
// row's top K to the log-probability and lse, which it computes with the same code as jk_xout_logprob's combine.
#include "split_tma.cuh"
#include "../../include/jkb200.h"
#include <algorithm>

using namespace jk;

namespace {

constexpr int kBN = 128, kBK = 64, kS = 3;
constexpr int kWsHead = 256;                      // workspace: status word, then the pairs, the target logits, a pad

struct ScoreP {
    const long long* targets;
    float2* part;                                 // [M][n_bt] (max, sum exp)
    float* tlogit;                                // [M]
    unsigned* status;
    int M, bins, n_kb, n_bt;
};

// the statistics epilogue's extra workspace (jk_xout_stats)
struct StatsP {
    float* u;                                     // [M][n_bt] sum (z - max) exp(z - max)
    float* topv;                                  // [M][n_bt][k] the tile's k largest logits, descending
    int* topi;                                    // [M][n_bt][k] their bins (ties: lower bin first; -1 past the tile)
    int k;
};

// the k largest logits of one row of a tile (the four lanes of a quad, columns c0 + 8 i + e of acc[4 i + 2 h + e]) by
// k rounds of argmax over what is not yet taken, ties to the lower bin; lane 0 of the quad writes them
__device__ __forceinline__ void tile_topk(const float (&acc)[kBN / 2], int h, const ScoreP& P, const StatsP& S, int r,
                                          int bt, int c0, int lane) {
    const bool writer = (lane & 3) == 0 && r < P.M;
    const size_t slot = (size_t)r * P.n_bt + bt;
    uint32_t taken = 0;
    for (int j = 0; j < S.k; ++j) {
        float bv = -INFINITY;
        int bc = -1;
#pragma unroll
        for (int i = 0; i < kBN / 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = c0 + 8 * i + e;
                const float z = acc[4 * i + 2 * h + e] * kWInv;
                if (col < P.bins && !((taken >> (2 * i + e)) & 1u) && (bc < 0 || z > bv)) { bv = z; bc = col; }
            }
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oc = __shfl_xor_sync(0xffffffffu, bc, o);
            if (oc >= 0 && (bc < 0 || ov > bv || (ov == bv && oc < bc))) { bv = ov; bc = oc; }
        }
        if (bc >= 0) {
            const int cc = bc & (kBN - 1);
            if ((lane & 3) == ((cc & 7) >> 1)) taken |= 1u << (2 * (cc >> 3) + (cc & 1));
        }
        if (writer) {
            S.topv[slot * S.k + j] = bv;
            S.topi[slot * S.k + j] = bc;
        }
    }
}

// the head on the streamed-weight pipeline (split_tma.cuh): an item is (128 rows x 128 bins), a K block the fp32
// activations [128 x 64] and the hi / lo x_out rows [128 x 64] of its bin tile
template <bool kStats>
struct HeadJob {
    using Ring = StreamRing<kBN, kS>;                        // 3 stages of 64 KB
    static constexpr bool kCheck = true, relu = false;
    const CUtensorMap *map_a, *map_w;                        // activations [rows, W] fp32, the split x_out
    ScoreP P;
    StatsP S;
    int n_kb, bins_pad;
    struct Tile { int mt, bt; };

    __device__ __forceinline__ unsigned* status() const { return P.status; }

    __device__ __forceinline__ Tile tile(int item) const {
        const int mt = item / P.n_bt, bt = item - mt * P.n_bt;
        return {mt, bt};
    }
    __device__ __forceinline__ void load(uint8_t* st, const Tile& t, int kb, uint64_t* bar) const {
        tma_load_2d(st, map_a, kb * kBK, t.mt * kBM, bar);          // rows >= M arrive as zeros
        tma_load_2d(st + Ring::kA, map_w, kb * kBK, t.bt * kBN, bar);
        tma_load_2d(st + Ring::kA + Ring::kB, map_w, kb * kBK, bins_pad + t.bt * kBN, bar);
    }
    // ---- per row: (max, sum exp) over this tile's bins, and the target's logit where it falls here.  The four lanes of
    // a quad hold the tile's 128 columns of two rows (d[4 i + 2 h + e]: row + 8 h, column 8 i + 2 (lane % 4) + e); they
    // combine in a fixed shuffle order ----
    __device__ __forceinline__ void epilogue(const float (&acc)[kBN / 2], const Tile& t, int rq, int lane) const {
        const int c0 = t.bt * kBN + 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = t.mt * kBM + rq + 8 * h;
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < kBN / 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (c0 + 8 * i + e < P.bins) mx = fmaxf(mx, acc[4 * i + 2 * h + e] * kWInv);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const long long tg = r < P.M && (!kStats || P.targets) ? __ldg(P.targets + r) : -1;
            float se = 0.f, u = 0.f;
#pragma unroll
            for (int i = 0; i < kBN / 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = c0 + 8 * i + e;
                    if (col < P.bins) {
                        const float z = acc[4 * i + 2 * h + e] * kWInv;
                        if constexpr (kStats) {
                            const float ex = expf(z - mx);
                            se += ex;
                            u += (z - mx) * ex;
                        } else {
                            se += expf(z - mx);
                        }
                        if (col == tg) P.tlogit[r] = z;
                    }
                }
            se += __shfl_xor_sync(0xffffffffu, se, 1);
            se += __shfl_xor_sync(0xffffffffu, se, 2);
            if ((lane & 3) == 0 && r < P.M) P.part[(size_t)r * P.n_bt + t.bt] = make_float2(mx, se);
            if constexpr (kStats) {
                u += __shfl_xor_sync(0xffffffffu, u, 1);
                u += __shfl_xor_sync(0xffffffffu, u, 2);
                if ((lane & 3) == 0 && r < P.M) S.u[(size_t)r * P.n_bt + t.bt] = u;
                if (S.k) tile_topk(acc, h, P, S, r, t.bt, c0, lane);
            }
        }
    }
};

template <bool kStats>
__global__ void __launch_bounds__(kStreamThreads, 1)
xout_head_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_w, ScoreP P,
                 StatsP S, int total_items) {
    extern __shared__ __align__(1024) uint8_t sm_raw[];
    const HeadJob<kStats> job{&map_h, &map_w, P, S, P.n_kb, P.n_bt * kBN};
    streamed_pipeline(job, sm_raw, total_items);
}

// one thread per row: the row's pairs in bin-tile order -> lse, logp.  Status bit 0: an activation outside the fp16
// split's range (every row is void); bit 1: a target outside [0, bins)
// lse of a row from its (max, sum exp) pairs in bin-tile order; mx gets the row max.  Both combines use it, so that
// jk_xout_stats gives jk_xout_logprob's lse and logp bit for bit
__device__ __forceinline__ float row_lse(const float2* p, int n_bt, float& mx) {
    mx = -INFINITY;
    for (int j = 0; j < n_bt; ++j) mx = fmaxf(mx, p[j].x);
    float se = 0.f;
    for (int j = 0; j < n_bt; ++j) se += p[j].y * expf(p[j].x - mx);
    return mx + logf(se);
}

__global__ void xout_combine_kernel(ScoreP P, float* __restrict__ logp, float* __restrict__ lse) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= P.M) return;
    const float2* p = P.part + (size_t)r * P.n_bt;
    float mx;
    const float l = row_lse(p, P.n_bt, mx);
    const long long tg = P.targets[r];
    const bool tg_ok = tg >= 0 && tg < P.bins;
    if (!tg_ok) atomicOr(P.status, 2u);
    const bool ok = tg_ok && (*reinterpret_cast<volatile unsigned*>(P.status) & 1u) == 0;
    logp[r] = ok ? P.tlogit[r] - l : __int_as_float(0x7fffffff);
    if (lse) lse[r] = ok ? l : __int_as_float(0x7fffffff);
}

constexpr int kStatsCombineThreads = 128;

// one thread per row, as xout_combine_kernel, and further:
//   entropy H = lse - sum p z = log S - (1/S) sum_j w_j (u_j + (m_j - m) s_j),  w_j = exp(m_j - m),  S = sum_j w_j s_j
//   in fp64 over the tiles' (m_j, s_j, u_j) rescaled to the row max m;
//   the row's top k: the tiles' lists merged in bin-tile order by insertion into a sorted list in shared memory (a
//   later tile's equal logit has the higher bin, so it goes behind), written as bins and logit - lse.
// Targets may be absent (NULL); a void row (bit 0, or its target out of range) gets nan and id -1 everywhere.
__global__ void __launch_bounds__(kStatsCombineThreads)
xout_stats_combine_kernel(ScoreP P, StatsP S, float* __restrict__ logp, float* __restrict__ entropy,
                          long long* __restrict__ topk_ids, float* __restrict__ topk_logp, float* __restrict__ lse) {
    extern __shared__ float2 lst[];               // [k][kStatsCombineThreads] (logit, bin as int bits)
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= P.M) return;
    const float2* p = P.part + (size_t)r * P.n_bt;
    float mx;
    const float l = row_lse(p, P.n_bt, mx);
    bool ok = true;
    if (P.targets) {
        const long long tg = P.targets[r];
        if (!(tg >= 0 && tg < P.bins)) { ok = false; atomicOr(P.status, 2u); }
    }
    ok = ok && (*reinterpret_cast<volatile unsigned*>(P.status) & 1u) == 0;
    const float nan = __int_as_float(0x7fffffff);
    if (P.targets) logp[r] = ok ? P.tlogit[r] - l : nan;
    if (lse) lse[r] = ok ? l : nan;
    const float* u = S.u + (size_t)r * P.n_bt;
    double sw = 0.0, a = 0.0;
    for (int j = 0; j < P.n_bt; ++j) {
        const double dm = (double)p[j].x - (double)mx, w = exp(dm);
        sw += w * (double)p[j].y;
        a += w * ((double)u[j] + dm * (double)p[j].y);
    }
    entropy[r] = ok ? (float)(log(sw) - a / sw) : nan;
    if (S.k == 0) return;
    float2* L = lst + threadIdx.x;
    const int K = S.k;
    int n = 0;
    for (int j = 0; j < P.n_bt; ++j) {
        const size_t slot = ((size_t)r * P.n_bt + j) * K;
        for (int c = 0; c < K; ++c) {
            const int id = S.topi[slot + c];
            const float v = S.topv[slot + c];
            if (id < 0 || (n == K && !(v > L[(K - 1) * kStatsCombineThreads].x))) break;   // the tile's list is sorted
            int q = n < K ? n++ : K - 1;
            for (; q > 0; --q) {
                const float2 prev = L[(q - 1) * kStatsCombineThreads];
                if (!(v > prev.x || (v == prev.x && id < __float_as_int(prev.y)))) break;
                L[q * kStatsCombineThreads] = prev;
            }
            L[q * kStatsCombineThreads] = make_float2(v, __int_as_float(id));
        }
    }
    for (int q = 0; q < K; ++q) {
        const float2 e = L[q * kStatsCombineThreads];
        const bool have = ok && q < n;
        if (topk_ids) topk_ids[(size_t)r * K + q] = have ? __float_as_int(e.y) : -1;
        if (topk_logp) topk_logp[(size_t)r * K + q] = have ? e.x - l : nan;
    }
}

// x_out [bins, W] fp32 -> [hi | lo][bins_pad][W] fp16 of 2^8 w (padding rows stay as the caller zeroed them)
__global__ void pack_xout_split_kernel(const float* __restrict__ w, unsigned short* __restrict__ split, int bins, int bins_pad,
                                       int W, unsigned* status) {
    const long long total = (long long)bins * W;
    bool ok = true;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        __half h, l;
        const float v = kWScale * __ldg(w + i);
        ok &= fabsf(v) <= kF16Max;
        split_f16(v, h, l);
        split[i] = __half_as_ushort(h);
        split[(size_t)bins_pad * W + i] = __half_as_ushort(l);
    }
    if (!ok) atomicOr(status, 1u);
}

int n_bin_tiles(int bins) { return (bins + kBN - 1) / kBN; }
size_t split_plane_bytes(int bins, int W) { return (size_t)n_bin_tiles(bins) * kBN * W * 2; }
size_t pad_bytes(int W) { return (size_t)kBM * W * 4; }
size_t up256(size_t b) { return (b + 255) / 256 * 256; }
// workspace: status head | pairs | target logits | (stats: u | top-k logits | top-k bins) | zero-padded rows if M < 128
size_t stats_bytes(int M, int bins, int k) {
    const size_t slots = (size_t)M * n_bin_tiles(bins);
    return up256(slots * 4) + 2 * up256(slots * k * 4);
}
size_t ws_bytes(int M, int W, int bins) {
    const size_t pairs = ((size_t)M * n_bin_tiles(bins) * 8 + 255) / 256 * 256, tl = ((size_t)M * 4 + 255) / 256 * 256;
    return kWsHead + pairs + tl + (M < kBM ? pad_bytes(W) : 0);
}

int read_status(const unsigned* status, unsigned* out, cudaStream_t stream) {
    JK_CHECK_CUDA(cudaMemcpyAsync(out, status, sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
    JK_CHECK_CUDA(cudaStreamSynchronize(stream));
    return 0;
}

// P's pointers into the workspace, the status cleared, and xout_head_kernel<kStats> launched on the tiles of h
template <bool kStats>
int launch_head(const float* h, int m, int width, const void* w_split, int bins, const int64_t* targets, char* ws,
                size_t need, ScoreP& P, const StatsP& S, cudaStream_t stream) {
    constexpr int kSmem = HeadJob<kStats>::Ring::smem;
    const int n_bt = n_bin_tiles(bins), bins_pad = n_bt * kBN;
    const long long total = (long long)((m + kBM - 1) / kBM) * n_bt;
    JK_REQUIRE(total < (1ll << 31), "too many rows");
    P.status = reinterpret_cast<unsigned*>(ws);
    P.part = reinterpret_cast<float2*>(ws + kWsHead);
    P.tlogit = reinterpret_cast<float*>(ws + kWsHead + ((size_t)m * n_bt * 8 + 255) / 256 * 256);
    P.targets = reinterpret_cast<const long long*>(targets);
    P.M = m; P.bins = bins; P.n_kb = width / kBK; P.n_bt = n_bt;
    JK_CHECK_CUDA(cudaMemsetAsync(P.status, 0, sizeof(unsigned), stream));
    // fewer rows than one tile: the tile is staged from a zero-padded copy, so the tensor map never has a box larger
    // than the tensor
    const float* hsrc = h;
    int rows = m;
    if (m < kBM) {
        float* pad = reinterpret_cast<float*>(ws + need - pad_bytes(width));
        JK_CHECK_CUDA(cudaMemsetAsync(pad, 0, pad_bytes(width), stream));
        JK_CHECK_CUDA(cudaMemcpyAsync(pad, h, (size_t)m * width * 4, cudaMemcpyDeviceToDevice, stream));
        hsrc = pad;
        rows = kBM;
    }
    CUtensorMap map_h, map_w;
    {
        const cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)rows};
        const cuuint64_t strides[1] = {(cuuint64_t)width * 4};
        const cuuint32_t box[2] = {kBK, kBM};
        if (int rc = encode_tensor_map(&map_h, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, hsrc, dims, strides, box,
                                       CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
            return rc;
    }
    {
        const cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)2 * bins_pad};
        const cuuint64_t strides[1] = {(cuuint64_t)width * 2};
        const cuuint32_t box[2] = {kBK, kBN};
        if (int rc = encode_tensor_map(&map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w_split, dims, strides, box,
                                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
            return rc;
    }
    int sms = 0;
    if (int rc = set_max_smem_once<xout_head_kernel<kStats>>(kSmem)) return rc;
    if (int rc = sm_count(&sms)) return rc;
    const unsigned grid = (unsigned)std::min<long long>(total, sms);
    xout_head_kernel<kStats><<<grid, kStreamThreads, kSmem, stream>>>(map_h, map_w, P, S, (int)total);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" int jk_xout_split_bytes(int bins, int width, size_t* bytes) {
    JK_REQUIRE(bytes, "null argument");
    JK_REQUIRE(bins >= 1 && width >= 64 && width % 64 == 0, "need bins >= 1 and width a positive multiple of 64 (got %d, %d)",
               bins, width);
    *bytes = 2 * split_plane_bytes(bins, width) + 16;    // + the status word of the range check
    return 0;
}

extern "C" int jk_pack_xout_split(const float* w, void* split, int bins, int width, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    size_t bytes = 0;
    if (int rc = jk_xout_split_bytes(bins, width, &bytes)) return rc;
    JK_REQUIRE(w && split, "null argument");
    JK_REQUIRE(((uintptr_t)split & 15) == 0, "split must be 16-byte aligned");
    unsigned* status = reinterpret_cast<unsigned*>(static_cast<char*>(split) + 2 * split_plane_bytes(bins, width));
    JK_CHECK_CUDA(cudaMemsetAsync(split, 0, bytes, stream));
    const long long total = (long long)bins * width;
    const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, 65535);
    pack_xout_split_kernel<<<blocks, 256, 0, stream>>>(w, static_cast<unsigned short*>(split), bins,
                                                       n_bin_tiles(bins) * kBN, width, status);
    JK_CHECK_CUDA(cudaGetLastError());
    unsigned st = 0;
    if (int rc = read_status(status, &st, stream)) return rc;
    JK_REQUIRE(st == 0, "x_out weight outside the 2^8-scaled fp16 split (|w| > %g or not finite)", kF16Max / kWScale);
    return 0;
}

extern "C" int jk_xout_logprob_workspace_bytes(int m, int width, int bins, size_t* bytes) {
    JK_REQUIRE(bytes, "null argument");
    JK_REQUIRE(m >= 0 && bins >= 1 && width >= 64 && width % 64 == 0,
               "need m >= 0, bins >= 1 and width a positive multiple of 64 (got %d, %d, %d)", m, bins, width);
    *bytes = ws_bytes(m, width, bins);
    return 0;
}

extern "C" int jk_xout_logprob(const float* h, int m, int width, const void* w_split, int bins, const int64_t* targets,
                               float* logp, float* lse, void* workspace, size_t workspace_bytes, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    size_t need = 0;
    if (int rc = jk_xout_logprob_workspace_bytes(m, width, bins, &need)) return rc;
    JK_REQUIRE(h && w_split && targets && logp && workspace, "null argument");
    JK_REQUIRE(workspace_bytes >= need, "workspace of %zu bytes, need %zu", workspace_bytes, need);
    JK_REQUIRE(((uintptr_t)h & 15) == 0 && ((uintptr_t)w_split & 15) == 0 && ((uintptr_t)workspace & 255) == 0,
               "h and w_split must be 16-byte aligned, workspace 256-byte aligned");
    if (m == 0) return 0;
    ScoreP P;
    if (int rc = launch_head<false>(h, m, width, w_split, bins, targets, static_cast<char*>(workspace), need, P, StatsP{},
                                    stream))
        return rc;
    xout_combine_kernel<<<(m + 255) / 256, 256, 0, stream>>>(P, logp, lse);
    JK_CHECK_CUDA(cudaGetLastError());
    unsigned st = 0;
    if (int rc = read_status(P.status, &st, stream)) return rc;
    JK_REQUIRE((st & 1u) == 0, "an activation lies outside the fp16 split's range (|h| > 65504 or not finite)");
    JK_REQUIRE((st & 2u) == 0, "a target lies outside [0, %d)", bins);
    return 0;
}

extern "C" int jk_xout_stats_workspace_bytes(int m, int width, int bins, int k, size_t* bytes) {
    JK_REQUIRE(bytes, "null argument");
    JK_REQUIRE(m >= 0 && bins >= 1 && width >= 64 && width % 64 == 0,
               "need m >= 0, bins >= 1 and width a positive multiple of 64 (got %d, %d, %d)", m, bins, width);
    JK_REQUIRE(k >= 0 && k <= JK_XOUT_STATS_MAX_K && k <= bins, "need 0 <= k <= min(%d, bins) (got k %d, bins %d)",
               JK_XOUT_STATS_MAX_K, k, bins);
    *bytes = ws_bytes(m, width, bins) + stats_bytes(m, bins, k);
    return 0;
}

extern "C" int jk_xout_stats(const float* h, int m, int width, const void* w_split, int bins, const int64_t* targets,
                             int k, float* logp, float* entropy, int64_t* topk_ids, float* topk_logp, float* lse,
                             void* workspace, size_t workspace_bytes, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    size_t need = 0;
    if (int rc = jk_xout_stats_workspace_bytes(m, width, bins, k, &need)) return rc;
    JK_REQUIRE(h && w_split && entropy && workspace, "null argument");
    JK_REQUIRE(!targets == !logp, "targets and logp are given together or not at all");
    JK_REQUIRE(k == 0 || topk_ids || topk_logp, "k = %d but neither topk_ids nor topk_logp is given", k);
    JK_REQUIRE(workspace_bytes >= need, "workspace of %zu bytes, need %zu", workspace_bytes, need);
    JK_REQUIRE(((uintptr_t)h & 15) == 0 && ((uintptr_t)w_split & 15) == 0 && ((uintptr_t)workspace & 255) == 0,
               "h and w_split must be 16-byte aligned, workspace 256-byte aligned");
    if (m == 0) return 0;
    // the stats arrays sit between the logprob layout's target logits and its zero-padded rows
    char* ws = static_cast<char*>(workspace);
    const size_t slots = (size_t)m * n_bin_tiles(bins);
    char* sp = ws + ws_bytes(m, width, bins) - (m < kBM ? pad_bytes(width) : 0);
    StatsP S;
    S.u = reinterpret_cast<float*>(sp);
    S.topv = reinterpret_cast<float*>(sp + up256(slots * 4));
    S.topi = reinterpret_cast<int*>(sp + up256(slots * 4) + up256(slots * k * 4));
    S.k = k;
    ScoreP P;
    if (int rc = launch_head<true>(h, m, width, w_split, bins, targets, ws, need, P, S, stream)) return rc;
    const size_t lst = (size_t)kStatsCombineThreads * k * sizeof(float2);
    xout_stats_combine_kernel<<<(m + kStatsCombineThreads - 1) / kStatsCombineThreads, kStatsCombineThreads, lst,
                                stream>>>(P, S, logp, entropy, reinterpret_cast<long long*>(topk_ids), topk_logp, lse);
    JK_CHECK_CUDA(cudaGetLastError());
    unsigned st = 0;
    if (int rc = read_status(P.status, &st, stream)) return rc;
    JK_REQUIRE((st & 1u) == 0, "an activation lies outside the fp16 split's range (|h| > 65504 or not finite)");
    JK_REQUIRE((st & 2u) == 0, "a target lies outside [0, %d)", bins);
    return 0;
}
