// Prefill-shape Conv1D on the Hopper tensor cores: Y[M, N] = X[M, K] . W[K, N] + b  (fp16 in, fp32 accumulate in
// registers, fp16 out), M = n_samples * rows >= 128.
//
// Reference: Conv1D.forward (transformer/ops.py:83-101) at the shapes where it is compute bound - here
// `c_enc_kv(encoder_kv)` of the encoder-decoder attention layers (factored_attention.py:273-287,
// M = n * encoder_dims = 4096, K = 4800, N = 2400 for 5b_lyrics), computed once per window.
//
// Kernel anatomy (one 128 x 128 output tile per CTA, K walked in 64-element blocks):
//   warp 8      TMA producer : cp.async.bulk.tensor.2d of the X tile [128 x 64] and the W^T tile [128 x 64], both
//                              K-major with the 128-byte swizzle, into a 3-stage ring
//   warps 0-7   consumers    : two warpgroups, rows 0-63 and 64-127 of the tile; each issues
//                              wgmma.mma_async m64n128k16 (64 fp32 accumulators per thread), keeps one K block in
//                              flight and frees the previous stage when it retires; then + bias, round to fp16 and
//                              store (rows and columns beyond M, N are predicated off; TMA zero-fills
//                              out-of-bounds loads)
// W is supplied transposed ([N, K], K contiguous) - the engine packs it once at weight load - so both
// operands are K-major, the layout wgmma reads without a transpose bit.
#include "engine.cuh"
#include "split_tma.cuh"

using namespace jk;

namespace {

constexpr int BM = 128, BN = 128, BK = 64, STAGES = 3;   // 3 x 32 KB: two CTAs per SM, one's epilogue overlaps the other's main loop
constexpr int kTileBytes = BM * BK * 2;                  // 16 KB per operand tile
constexpr int kGemmThreads = 288;                        // two consumer warpgroups + one producer warp
constexpr int kGemmSmem = STAGES * 2 * kTileBytes + 1024 + 256;

// The decode kernel's epilogues (decode_engine.cu gemm_phase), same fp16 rounding points:
//   0  Conv1D output rounded once from the fp32 accumulator           (ops.py:83-96)
//   1  quick_gelu with the reference's three fp16 roundings           (ops.py:33-35)
//   2  residual add in fp16                                           (transformer.py:82-83)
__device__ __forceinline__ __half epilogue_value(float acc, float bias, float res, int epi) {
    const float y = h2f_round(acc + bias);
    if (epi == 1) {
        const float z = h2f_round(1.702f * y);
        const float sg = h2f_round(1.0f / (1.0f + expf(-z)));
        return __float2half_rn(y * sg);
    }
    if (epi == 2) return __float2half_rn(res + y);
    return __float2half_rn(y);
}

__global__ void __launch_bounds__(kGemmThreads, 2)
prefill_gemm_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                    const float* __restrict__ bias, const __half* __restrict__ res, __half* __restrict__ y, int M, int N,
                    int K, int epi) {
    extern __shared__ __align__(1024) uint8_t gsm[];
    uint8_t* tiles = gsm;                                               // [STAGES][A | B]
    uint64_t* full = reinterpret_cast<uint64_t*>(gsm + STAGES * 2 * kTileBytes);
    uint64_t* empty = full + STAGES;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int nkb = (K + BK - 1) / BK;       // a K tail reads zeros: TMA zero-fills both operands beyond K

    if (tid == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); }   // empty: one arrival per warpgroup
        mbar_fence_init();
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_x)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb % STAGES;
                mbar_wait(&empty[s], ((kb / STAGES) & 1) ^ 1);
                mbar_expect_tx(&full[s], 2 * kTileBytes);
                tma_load_2d(tiles + s * 2 * kTileBytes, &map_x, kb * BK, m0, &full[s]);
                tma_load_2d(tiles + s * 2 * kTileBytes + kTileBytes, &map_w, kb * BK, n0, &full[s]);
            }
        }
        return;
    }
    const int wg = warp >> 2, wt = tid & 127;                            // warpgroup: rows 64 wg .. 64 wg + 63
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % STAGES;
        mbar_wait(&full[s], (kb / STAGES) & 1);
        const uint32_t a0 = smem_u32(tiles + s * 2 * kTileBytes) + wg * (64 * 128), b0 = smem_u32(tiles + s * 2 * kTileBytes + kTileBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)                                // 16 fp16 = 32 bytes per MMA K step
            wgmma_ss<BN>(acc, wgmma_desc_sw128(a0 + k * 32), wgmma_desc_sw128(b0 + k * 32));
        wgmma_commit();
        wgmma_wait<1>();                                                 // block kb - 1 has retired: free its stage
        if (kb > 0 && wt == 0) mbar_arrive(&empty[(kb - 1) % STAGES]);
    }
    wgmma_wait<0>();

    const int r0 = m0 + wg * 64 + (wt >> 5) * 16 + (lane >> 2);
    const bool pairs = (N & 1) == 0;                                     // 4-byte aligned column pairs
#pragma unroll
    for (int j = 0; j < BN / 4; ++j) {                                   // j = 2 i + h: columns 8 i + .., row r0 + 8 h
        const int row = r0 + 8 * (j & 1), col = n0 + 8 * (j >> 1) + 2 * (lane & 3);
        const float v0 = acc[2 * j], v1 = acc[2 * j + 1];
        if (row < M) {
            __half* yr = y + (size_t)row * N;
            const __half* rr = res ? res + (size_t)row * N : nullptr;
            if (pairs && col + 1 < N) {
                const float2 bb = bias ? make_float2(bias[col], bias[col + 1]) : make_float2(0.f, 0.f);
                const float2 rv = epi == 2 ? __half22float2(*reinterpret_cast<const __half2*>(rr + col)) : make_float2(0.f, 0.f);
                *reinterpret_cast<__half2*>(yr + col) =
                    __halves2half2(epilogue_value(v0, bb.x, rv.x, epi), epilogue_value(v1, bb.y, rv.y, epi));
            } else {
                if (col < N) yr[col] = epilogue_value(v0, bias ? bias[col] : 0.f, epi == 2 ? __half2float(rr[col]) : 0.f, epi);
                if (col + 1 < N)
                    yr[col + 1] = epilogue_value(v1, bias ? bias[col + 1] : 0.f, epi == 2 ? __half2float(rr[col + 1]) : 0.f, epi);
            }
        }
    }
}

// 2-D fp16 row-major [rows, K] tensor, box = [128 rows x 64 columns], 128-byte swizzle, zero fill out of bounds
int make_map(CUtensorMap* map, const void* base, int rows, int K) {
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
    return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

}  // namespace

int jk::gemm_f16_tc(const void* x, const void* w_t, const float* bias, const void* res, void* y, int M, int N, int K,
                    int epi, cudaStream_t stream) {
    JK_REQUIRE(x && w_t && y, "null argument");
    JK_REQUIRE(M >= 1 && N >= 1 && K >= BK && K % 8 == 0, "prefill GEMM needs K >= %d and K %% 8 == 0 (16-byte rows for TMA); got M %d N %d K %d", BK, M, N, K);
    JK_REQUIRE((((uintptr_t)x | (uintptr_t)w_t | (uintptr_t)y | (uintptr_t)res) & 15) == 0, "operands must be 16-byte aligned");
    JK_REQUIRE(epi >= 0 && epi <= 2 && (epi != 2 || res), "bad epilogue %d (0, 1, or 2 with res)", epi);
    CUtensorMap mx, mw;
    int rc = make_map(&mx, x, M, K);
    if (rc) return rc;
    rc = make_map(&mw, w_t, N, K);
    if (rc) return rc;
    rc = set_max_smem_once<prefill_gemm_kernel>(kGemmSmem);
    if (rc) return rc;
    dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
    prefill_gemm_kernel<<<grid, kGemmThreads, kGemmSmem, stream>>>(mx, mw, bias, (const __half*)res, (__half*)y, M, N, K, epi);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_conv1d_prefill_f16(const void* x, const void* w_t, const float* bias, void* y, int M, int N, int K,
                                     jk_stream_t stream_) {
    return jk::gemm_f16_tc(x, w_t, bias, nullptr, y, M, N, K, 0, (cudaStream_t)stream_);
}

extern "C" int jk_prefill_gemm_f16(const void* x, const void* w_t, const float* bias, const void* res, void* y, int M, int N,
                                   int K, int epi, jk_stream_t stream_) {
    return jk::gemm_f16_tc(x, w_t, bias, res, y, M, N, K, epi, (cudaStream_t)stream_);
}
