// The split-precision format of the decoder-side tensor-core kernels (vqvae_kernels.cu, vqvae_t5.cu) and the x_out
// log-softmax (score.cu): a value v becomes hi = fp16(v), lo = fp16(v - hi) (22 significant bits, rounded to nearest,
// saturating at the fp16 range), and every product runs as hi.w_hi + lo.w_hi + hi.w_lo with fp32 accumulation.  Weights
// are scaled by kWScale before their split and the epilogues multiply by kWInv.  Also the TMA helpers of the kernels
// that stage fp32 activations with TMA and split them into hi / lo planes in shared memory.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace jk {

// 2^8: a typical |w| ~ 0.05 would have its fp16 remainder (~2e-5) in the subnormal range, where the split keeps only
// ~19 bits; the scaling is exact
constexpr float kWScale = 256.f, kWInv = 1.f / 256.f;

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
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// byte offset of 16-byte chunk j of row r inside a K-major 128-byte-swizzled plane
__device__ __forceinline__ uint32_t sw_off(int r, int j) { return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((j ^ (r & 7)) << 4)); }
__device__ __forceinline__ void named_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

typedef CUresult (*EncodeTiledFnT5)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFnT5 t5_encode() {
    static EncodeTiledFnT5 fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFnT5>(p);
    }
    return fn;
}

}  // namespace jk
