// The split-precision format of the decoder-side tensor-core kernels (vqvae_kernels.cu, vqvae_t5.cu) and the x_out
// log-softmax (score.cu): a value v becomes hi = fp16(v), lo = fp16(v - hi) (22 significant bits, rounded to nearest,
// saturating at the fp16 range), and every product runs as hi.w_hi + lo.w_hi + hi.w_lo with fp32 accumulation.  Weights
// are scaled by kWScale before their split and the epilogues multiply by kWInv.
//
// Also the machinery of the kernels that stage fp32 activations with TMA and split them into hi / lo planes in shared
// memory: the TMA helpers and the host's tensor-map encoder (also used by prefill_gemm.cu), the converter that splits a
// 128-row fp32 tile into swizzled planes, the three-product wgmma of one K block, and the streamed-weight pipeline that
// conv_wide_kernel (vqvae_t5.cu) and xout_head_kernel (score.cu) run.  The tap pipeline of resblock_t5_kernel and
// conv_t5_kernel, whose weights stay in shared memory, lives in vqvae_t5.cu.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace jk {

// 2^8: a typical |w| ~ 0.05 would have its fp16 remainder (~2e-5) in the subnormal range, where the split keeps only
// ~19 bits; the scaling is exact
constexpr float kWScale = 256.f, kWInv = 1.f / 256.f;
constexpr float kF16Max = 65504.f;
constexpr int kBM = 128;                  // rows (positions) of a tile = two wgmma M blocks of 64

// one value -> hi / lo fp16
__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
    unsigned short h, l;
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(v));
    hi = __ushort_as_half(h);
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(l) : "f"(v - __half2float(hi)));
    lo = __ushort_as_half(l);
}
// two values -> packed hi / lo fp16 pairs (a in the low half)
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
    float ha, hb;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
    asm("{\n\t.reg .f16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, h;\n\t}" : "=f"(ha), "=f"(hb) : "r"(hi));
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(b - hb), "f"(a - ha));
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// the dynamic shared-memory base rounded up to 1024 bytes: TMA's 128-byte swizzle needs 1024-byte aligned stages
__device__ __forceinline__ uint8_t* align_1024(uint8_t* p) { return p + ((1024u - (smem_u32(p) & 1023u)) & 1023u); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// byte offset of 16-byte chunk j of row r inside a K-major 128-byte-swizzled plane
__device__ __forceinline__ uint32_t sw_off(int r, int j) { return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((j ^ (r & 7)) << 4)); }
__device__ __forceinline__ void named_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// fp32 tile [128 rows][CH float4 chunks] at src -> (relu) -> hi plane at dst, lo plane at dst + 16 KB, in the K-major
// 128-byte-swizzled layout wgmma reads, by one group of 128 converter threads (ct = 0..127).
//   kInPlace: dst is src.  Every value is read into registers before the group's named barrier 1, so the planes can
//             overwrite the block they come from.  Without it there is no barrier (two groups may convert at once).
//   kCheck:   returns false if a value lies outside the fp16 range (|v| > 65504, inf, nan); otherwise returns true.
template <int CH, bool kInPlace, bool kCheck>
__device__ __forceinline__ bool convert_planes(const uint8_t* src, uint8_t* dst, int ct, bool relu) {
    constexpr int PER = kBM * CH / 128;                     // items per thread
    const float4* f = reinterpret_cast<const float4*>(src);
    float4 v[PER];
#pragma unroll
    for (int j = 0; j < PER; ++j) v[j] = f[ct + j * 128];
    uint2 h[PER], l[PER];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
        if (relu) { v[j].x = fmaxf(v[j].x, 0.f); v[j].y = fmaxf(v[j].y, 0.f); v[j].z = fmaxf(v[j].z, 0.f); v[j].w = fmaxf(v[j].w, 0.f); }
        if constexpr (kCheck)
            ok &= fabsf(v[j].x) <= kF16Max && fabsf(v[j].y) <= kF16Max && fabsf(v[j].z) <= kF16Max && fabsf(v[j].w) <= kF16Max;
        split_f16x2(v[j].x, v[j].y, h[j].x, l[j].x);
        split_f16x2(v[j].z, v[j].w, h[j].y, l[j].y);
    }
    if constexpr (kInPlace) named_sync(1);
#pragma unroll
    for (int j = 0; j < PER; ++j) {
        const int item = ct + j * 128, r = item / CH, c4 = item % CH;
        const uint32_t o = sw_off(r, c4 >> 1) + (c4 & 1) * 8;
        *reinterpret_cast<uint2*>(dst + o) = h[j];
        *reinterpret_cast<uint2*>(dst + kBM * 128 + o) = l[j];
    }
    return ok;
}

// one K block of CI channels: CI / 16 k-steps x 3 products (lo.w_hi, hi.w_lo, hi.w_hi) of this warpgroup's 64 rows
template <int CI, int CO>
__device__ __forceinline__ void mma_tap(float (&acc)[CO / 2], uint32_t ah, uint32_t al, uint32_t bh, uint32_t bl) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < CI / 16; ++k) {
        wgmma_ss<CO>(acc, wgmma_desc_sw128(al + k * 32), wgmma_desc_sw128(bh + k * 32));
        wgmma_ss<CO>(acc, wgmma_desc_sw128(ah + k * 32), wgmma_desc_sw128(bl + k * 32));
        wgmma_ss<CO>(acc, wgmma_desc_sw128(ah + k * 32), wgmma_desc_sw128(bh + k * 32));
    }
    wgmma_commit();
}

// ---------------------------------------------------------------------------------------
// The streamed-weight pipeline: 512 threads, one persistent CTA per SM, work items of 128 rows x BN columns whose
// K runs in 64-channel blocks through an S-stage ring.  A stage holds the fp32 activation block [128 x 64] as TMA
// delivers it - the converters turn it IN PLACE into its hi / lo fp16 planes (16 KB each) - and the hi / lo planes of
// the weight block [BN x 64], which TMA loads with the 128-byte swizzle from a weight split once per weight load.
// ---------------------------------------------------------------------------------------
template <int BN, int S>
struct StreamRing {
    static constexpr int kBN = BN, kS = S;
    static constexpr int kA = kBM * 64 * 4;                  // fp32 block; after conversion hi plane | lo plane
    static constexpr int kAPlane = kBM * 128;
    static constexpr int kB = BN * 128;                      // one weight plane: BN rows x 64 fp16
    static constexpr int kStage = kA + 2 * kB;
    static constexpr int offBar = kS * kStage;
    static constexpr int smem = offBar + 128 + 1024;         // barriers, and slack to align the ring to 1024 bytes
};
constexpr int kStreamThreads = 512;

// Roles, four warpgroups, connected by mbarriers only:
//   warp 12      TMA producer: J.load puts K block kb of an item into a stage (warps 13-15 only hand their registers back);
//   warps 8-11   converters: fp32 block -> (relu) -> hi / lo planes in place; with Job::kCheck a value outside the fp16
//                range sets bit 0 of *J.status instead of saturating;
//   warps 0-7    consumers, rows 0-63 / 64-127 of the item: every K block's 12 wgmmas go into a zeroed partial that is then
//                added to the item's fp32 sum with ordinary (round-to-nearest) adds.  The tensor core's own accumulation
//                rounds each k16 step's sum towards zero, and over long K that bias grows to ~2e-5 of the output scale;
//                promoted every 64 channels it stays at the exact kernel's level.  Then J.epilogue on the sum.
// The Job supplies Ring (a StreamRing), kCheck (and status() if set), relu, map_a / map_w (prefetched), n_kb, tile(item)
// (an item's tile coordinates), load(stage, tile, kb, bar) and epilogue(acc, tile, rq, lane) (rq: the thread's first
// accumulator row in the item).
template <class Job>
__device__ __forceinline__ void streamed_pipeline(const Job& J, uint8_t* sm_raw, int total_items) {
    using L = typename Job::Ring;
    constexpr int S = L::kS, BN = L::kBN;
    uint8_t* sm = align_1024(sm_raw);
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + L::offBar);
    uint64_t *full = bars, *conv = bars + S, *empty = bars + 2 * S;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        // full: the producer's expect_tx (activation + weight bytes); conv: the 128 converter threads; empty: one arrival
        // per consumer warpgroup once its MMAs on the stage have retired
        for (int i = 0; i < S; ++i) { mbar_init(&full[i], 1); mbar_init(&conv[i], 128); mbar_init(&empty[i], 2); }
        mbar_fence_init();
        prefetch_tensormap(J.map_a);
        prefetch_tensormap(J.map_w);
    }
    __syncthreads();
    const int first = blockIdx.x, stride = gridDim.x;

    // register reallocation (setmaxnreg, whole warpgroups): the block launches with 128 per thread (65536 / 512);
    // 2 x 128 x 184 + 128 x 104 + 128 x 40 = 65536
    if (warp >= 12) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 12 && lane == 0) {
            uint32_t kt = 0;
            for (int item = first; item < total_items; item += stride) {
                const auto t = J.tile(item);
                for (int kb = 0; kb < J.n_kb; ++kb, ++kt) {
                    const int s = kt % S;
                    mbar_wait(&empty[s], ((kt / S) & 1) ^ 1);
                    mbar_expect_tx(&full[s], (uint32_t)L::kStage);
                    J.load(sm + s * L::kStage, t, kb, &full[s]);
                }
            }
        }
    } else if (warp >= 8) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 104;");
        const int ct = tid & 127;
        bool ok = true;
        uint32_t kt = 0;
        for (int item = first; item < total_items; item += stride) {
            for (int kb = 0; kb < J.n_kb; ++kb, ++kt) {
                const int s = kt % S;
                mbar_wait(&full[s], (kt / S) & 1);
                uint8_t* st = sm + s * L::kStage;
                ok &= convert_planes<16, true, Job::kCheck>(st, st, ct, J.relu);
                fence_async_smem();                   // the planes are read by the tensor core (async proxy)
                mbar_arrive(&conv[s]);
            }
        }
        if constexpr (Job::kCheck)
            if (!ok) atomicOr(J.status(), 1u);
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 184;");
        const int wg = warp >> 2, wt = tid & 127, rq = wg * 64 + (wt >> 5) * 16 + (lane >> 2);
        const uint32_t ring = smem_u32(sm);
        uint32_t kt = 0;
        for (int item = first; item < total_items; item += stride) {
            const auto t = J.tile(item);
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            for (int kb = 0; kb < J.n_kb; ++kb, ++kt) {
                const int s = kt % S;
                const uint32_t ph = (kt / S) & 1;
                mbar_wait(&full[s], ph);              // weight planes (TMA)
                mbar_wait(&conv[s], ph);              // activation planes (converters)
                const uint32_t st = ring + s * L::kStage, ah = st + wg * (64 * 128), al = ah + L::kAPlane;
                float part[BN / 2];
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) part[i] = 0.f;
                mma_tap<64, BN>(part, ah, al, st + L::kA, st + L::kA + L::kB);
                wgmma_wait<0>();
                if (wt == 0) mbar_arrive(&empty[s]);  // the block has retired: free its stage
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
            }
            J.epilogue(acc, t, rq, lane);
        }
    }
}

// ---- host: tensor maps ----------------------------------------------------------------
// A tiled tensor map of the rank-dimensional tensor at base (dims and box innermost first, the byte strides of
// dimensions 1 .. rank - 1); no interleave, and out-of-bounds elements read as zeros
inline int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType type, int rank, const void* base, const cuuint64_t* dims,
                             const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle,
                             CUtensorMapL2promotion l2) {
    typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                      const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static const EncodeTiledFn enc = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
                        q == cudaDriverEntryPointSuccess;
        return ok ? reinterpret_cast<EncodeTiledFn>(p) : nullptr;
    }();
    JK_REQUIRE(enc, "cuTensorMapEncodeTiled is not available from the driver");
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUresult r = enc(map, type, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char shape[96];
        int n = 0;
        for (int d = rank - 1; d >= 0; --d)
            n += snprintf(shape + n, sizeof(shape) - n, d == rank - 1 ? "%llu" : ", %llu", (unsigned long long)dims[d]);
        JK_REQUIRE(false, "cuTensorMapEncodeTiled failed (%d) for a [%s] %s tensor", (int)r, shape,
                   type == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? "fp32" : "fp16");
    }
    return 0;
}
// fp32 activations [n, T, C] as the tensor [C, T, n] in box [box_c x 128 x 1], so that rows outside [0, T) of a clip
// arrive as zeros
inline int encode_rows_map(CUtensorMap* map, const float* x, int n, long long T, int C, int box_c) {
    const cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)T, (cuuint64_t)n};
    const cuuint64_t strides[2] = {(cuuint64_t)C * 4, (cuuint64_t)T * C * 4};
    const cuuint32_t box[3] = {(cuuint32_t)box_c, (cuuint32_t)kBM, 1};
    return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, x, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

}  // namespace jk
