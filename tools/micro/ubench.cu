// Micro-benchmarks that inform the decode-engine design: legacy HMMA latency/throughput,
// ldmatrix latency, L2 load latency (hit / written-by-another-SM), grid barrier round trip.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include <stdio.h>
#include <stdint.h>

__device__ __forceinline__ void mma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

template <int CHAINS>
__global__ void hmma_kernel(float* out, long long* cyc, int iters) {
    float c[CHAINS][4];
    for (int j = 0; j < CHAINS; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.f;
    uint32_t a = 0x3c003c00u + threadIdx.x, b = 0x3c003c00u;
    __syncthreads();
    long long t0 = clock64();
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < CHAINS; ++j) mma(c[j], a, a, a, a, b, b);
    }
    long long t1 = clock64();
    float s = 0;
    for (int j = 0; j < CHAINS; ++j) s += c[j][0] + c[j][1] + c[j][2] + c[j][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) cyc[0] = t1 - t0;
}

__global__ void chase_kernel(const int* p, int n, long long* cyc, int* sink) {
    int idx = 0;
    long long t0 = clock64();
    for (int i = 0; i < n; ++i) idx = __ldcg(p + idx);
    long long t1 = clock64();
    cyc[0] = t1 - t0;
    sink[0] = idx;
}

// block 0 writes a line, signals; block 1 (another SM) waits for the flag then times a load of that line
__global__ void pingpong_kernel(volatile int* flag, int* data, long long* cyc, int rounds) {
    if (blockIdx.x == 0) {
        for (int r = 1; r <= rounds; ++r) {
            data[threadIdx.x] = r;
            __syncthreads();
            if (threadIdx.x == 0) { __threadfence(); atomicExch((int*)flag, r); }
            while (*(flag + 32) < r) {}
            __syncthreads();
        }
    } else if (blockIdx.x == 1) {
        long long tot = 0;
        for (int r = 1; r <= rounds; ++r) {
            if (threadIdx.x == 0) {
                while (*flag < r) {}
                long long t0 = clock64();
                int v = __ldcg(data + 5);
                if (v != r) tot += 1000000;
                long long t1 = clock64();
                tot += t1 - t0;
                __threadfence();
                *(flag + 32) = r;
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) cyc[0] = tot / rounds;
    }
}

__global__ void gridbar_kernel(unsigned* bar, long long* cyc, int rounds) {
    long long t0 = clock64();
    for (int r = 1; r <= rounds; ++r) {
        __syncthreads();
        if (threadIdx.x == 0) {
            asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(bar), "r"(1u) : "memory");
            unsigned target = r * gridDim.x, v;
            do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory"); } while ((int)(v - target) < 0);
        }
        __syncthreads();
    }
    long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) cyc[0] = (t1 - t0) / rounds;
}

__global__ void bcast_read_kernel(const uint4* src, int n16, uint4* sink, long long* cyc) {
    // every CTA reads the same n16*16 bytes (activation broadcast pattern), 16 loads in flight per thread
    extern __shared__ uint4 sm4[];
    uint4* sm = sm4;
    __syncthreads();
    long long t0 = clock64();
    for (int i = threadIdx.x; i < n16; i += blockDim.x) sm[i] = __ldcg(src + i);
    __syncthreads();
    long long t1 = clock64();
    if (threadIdx.x == 0) { cyc[blockIdx.x] = t1 - t0; sink[blockIdx.x] = sm[(int)(t1 & 15)]; }
}

// replica of the decode GEMM inner loop: 8 warps split 128 k-steps, A via ldmatrix from a padded
// [16][K+8] tile, B fragments via LDS.64 from 16 KB slots, m16n8k16 HMMA, ncg column groups
__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
template <int MODE>
__global__ void gemm_loop_kernel(float* out, long long* cyc, int K, int ncg, int reps) {
    extern __shared__ uint4 sm4[];
    uint8_t* sm = reinterpret_cast<uint8_t*>(sm4);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int astride = (K + 8) * 2;
    uint8_t* acts = sm;
    uint8_t* wts = sm + 16 * astride;
    for (int i = tid; i < (16 * astride + 65536) / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(sm)[i] = 0x3c003c00u;
    __syncthreads();
    float acc[8][4];
    for (int j = 0; j < 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    const uint32_t arow = (uint32_t)__cvta_generic_to_shared(acts + (lane & 15) * astride + (lane >> 4) * 16);
    const int nkk = K >> 4;
    long long t0 = clock64();
    for (int rep = 0; rep < reps; ++rep) {
#pragma unroll 2
        for (int i = warp; i < nkk; i += 8) {
            uint32_t a[4];
            if (MODE == 0) ldsm4(a, arow + i * 32);
            else if (MODE == 1) {
                const uint8_t* ap = acts + (lane >> 2) * astride + (lane & 3) * 4 + i * 32;
                a[0] = *reinterpret_cast<const uint32_t*>(ap);
                a[1] = *reinterpret_cast<const uint32_t*>(ap + 8 * astride);
                a[2] = *reinterpret_cast<const uint32_t*>(ap + 16);
                a[3] = *reinterpret_cast<const uint32_t*>(ap + 8 * astride + 16);
            } else { a[0] = a[1] = a[2] = a[3] = 0x3c003c00u + i; }
            const uint2* bp = reinterpret_cast<const uint2*>(wts + (size_t)((i % 64) * ncg) * 256) + lane;
            uint2 bf[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) bf[j] = (j < ncg) ? bp[j * 32] : make_uint2(0, 0);
#pragma unroll
            if (MODE != 3) {
#pragma unroll
                for (int j = 0; j < 8; ++j) if (j < ncg) mma(acc[j], a[0], a[1], a[2], a[3], bf[j].x, bf[j].y);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) if (j < ncg) acc[j][0] += __uint_as_float(a[0] ^ bf[j].x) + __uint_as_float(a[3] ^ bf[j].y);
            }
        }
    }
    long long t1 = clock64();
    float s = 0; for (int j = 0; j < 8; ++j) s += acc[j][0] + acc[j][3];
    out[blockIdx.x * blockDim.x + tid] = s;
    if (tid == 0 && blockIdx.x == 0) cyc[0] = (t1 - t0) / reps;
}

__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
template <int NCG, int UNR>
__global__ void gemm_loop_t_kernel(float* out, long long* cyc, int K, int reps) {
    extern __shared__ uint4 sm4[];
    uint8_t* sm = reinterpret_cast<uint8_t*>(sm4);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int astride = (K + 8) * 2;
    for (int i = tid; i < (16 * astride + 65536) / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(sm)[i] = 0x3c003c00u;
    __syncthreads();
    float acc[NCG][4];
    for (int j = 0; j < NCG; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    const uint32_t arow = (uint32_t)__cvta_generic_to_shared(sm + (lane & 15) * astride + (lane >> 4) * 16);
    const uint32_t wbase = (uint32_t)__cvta_generic_to_shared(sm + 16 * astride) + lane * 8;
    const int nkk = K >> 4;
    long long t0 = clock64();
    for (int rep = 0; rep < reps; ++rep) {
#pragma unroll UNR
        for (int i = warp; i < nkk; i += 8) {
            uint32_t a[4];
            asm("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"(arow + i * 32));
            uint2 bf[NCG];
#pragma unroll
            for (int j = 0; j < NCG; ++j) bf[j] = lds64(wbase + (((i & 63) * NCG + j) << 8));
#pragma unroll
            for (int j = 0; j < NCG; ++j)
                asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                    : "+f"(acc[j][0]), "+f"(acc[j][1]), "+f"(acc[j][2]), "+f"(acc[j][3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(bf[j].x), "r"(bf[j].y));
        }
    }
    long long t1 = clock64();
    float s = 0; for (int j = 0; j < NCG; ++j) s += acc[j][0] + acc[j][3];
    out[blockIdx.x * blockDim.x + tid] = s;
    if (tid == 0 && blockIdx.x == 0) cyc[0] = (t1 - t0) / reps;
}

int main() {
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    int sms = prop.multiProcessorCount;
    printf("device %s, %d SMs, clock %d kHz\n", prop.name, sms, prop.clockRate);
    float* out; long long* cyc; cudaMalloc(&out, 1 << 24); cudaMallocManaged(&cyc, 4096 * 8);
    const int it = 4096;
    for (int warps : {1, 2, 4, 8}) {
        hmma_kernel<1><<<sms, 32 * warps>>>(out, cyc, it); cudaDeviceSynchronize();
        double c1 = (double)cyc[0] / it;
        hmma_kernel<2><<<sms, 32 * warps>>>(out, cyc, it); cudaDeviceSynchronize();
        double c2 = (double)cyc[0] / it / 2;
        hmma_kernel<4><<<sms, 32 * warps>>>(out, cyc, it); cudaDeviceSynchronize();
        double c4 = (double)cyc[0] / it / 4;
        hmma_kernel<8><<<sms, 32 * warps>>>(out, cyc, it); cudaDeviceSynchronize();
        double c8 = (double)cyc[0] / it / 8;
        printf("HMMA.16816.F32 %d warps/SM: cycles per HMMA per warp with 1/2/4/8 independent chains: %.1f %.1f %.1f %.1f\n", warps, c1, c2, c4, c8);
    }
    {
        int K = 2048, smem = 16 * (K + 8) * 2 + 65536, ncg = 2;
        cudaFuncSetAttribute(gemm_loop_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(gemm_loop_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(gemm_loop_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(gemm_loop_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        gemm_loop_kernel<0><<<sms, 256, smem>>>(out, cyc, K, ncg, 50); cudaDeviceSynchronize();
        printf("GEMM loop replica K=2048 ncg=2 256 thr, A via ldmatrix: %lld cycles  [%s]\n", cyc[0], cudaGetErrorString(cudaGetLastError()));
        gemm_loop_kernel<1><<<sms, 256, smem>>>(out, cyc, K, ncg, 50); cudaDeviceSynchronize();
        printf("   A via 4x LDS.32: %lld cycles\n", cyc[0]);
        gemm_loop_kernel<2><<<sms, 256, smem>>>(out, cyc, K, ncg, 50); cudaDeviceSynchronize();
        printf("   A constant (no A loads): %lld cycles\n", cyc[0]);
        gemm_loop_kernel<3><<<sms, 256, smem>>>(out, cyc, K, ncg, 50); cudaDeviceSynchronize();
        printf("   ldmatrix but no HMMA: %lld cycles\n", cyc[0]);
        gemm_loop_kernel<0><<<1, 256, smem>>>(out, cyc, K, ncg, 50); cudaDeviceSynchronize();
        printf("   ldmatrix, ONE CTA on the chip: %lld cycles\n", cyc[0]);
        gemm_loop_kernel<0><<<sms, 32, smem>>>(out, cyc, K, ncg, 50); cudaDeviceSynchronize();
        printf("   ldmatrix, 1 warp per CTA (128 k-steps in one warp): %lld cycles\n", cyc[0]);
    }
    {
        int K = 2048, smem = 16 * (K + 8) * 2 + 65536;
        cudaFuncSetAttribute(gemm_loop_t_kernel<2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(gemm_loop_t_kernel<2, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(gemm_loop_t_kernel<1, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(gemm_loop_t_kernel<4, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        gemm_loop_t_kernel<2, 1><<<sms, 256, smem>>>(out, cyc, K, 50); cudaDeviceSynchronize();
        printf("templated NCG=2 unroll 1: %lld cycles [%s]\n", cyc[0], cudaGetErrorString(cudaGetLastError()));
        gemm_loop_t_kernel<2, 4><<<sms, 256, smem>>>(out, cyc, K, 50); cudaDeviceSynchronize();
        printf("templated NCG=2 unroll 4: %lld cycles\n", cyc[0]);
        gemm_loop_t_kernel<1, 4><<<sms, 256, smem>>>(out, cyc, K, 50); cudaDeviceSynchronize();
        printf("templated NCG=1 unroll 4: %lld cycles\n", cyc[0]);
        gemm_loop_t_kernel<4, 4><<<sms, 256, smem>>>(out, cyc, K, 50); cudaDeviceSynchronize();
        printf("templated NCG=4 unroll 4: %lld cycles\n", cyc[0]);
    }
    // pointer chase in L2 (4 MB footprint, stride 4 KB)
    {
        int n = 1 << 20; int* h = (int*)malloc(n * 4);
        for (int i = 0; i < n; ++i) h[i] = (i + 1024 + 17) % n;
        int* d; cudaMalloc(&d, n * 4); cudaMemcpy(d, h, n * 4, cudaMemcpyHostToDevice);
        int* sink; cudaMalloc(&sink, 64);
        chase_kernel<<<1, 1>>>(d, 2000, cyc, sink); cudaDeviceSynchronize();
        chase_kernel<<<1, 1>>>(d, 2000, cyc, sink); cudaDeviceSynchronize();
        printf("dependent ld.global.cg chain (L2 resident): %.0f cycles per load\n", (double)cyc[0] / 2000);
    }
    {
        int* flag; int* data; cudaMalloc(&flag, 1024); cudaMalloc(&data, 4096); cudaMemset(flag, 0, 1024);
        pingpong_kernel<<<2, 32>>>(flag, data, cyc, 200); cudaDeviceSynchronize();
        printf("load of a line just written by another SM (after flag): %lld cycles\n", cyc[0]);
    }
    {
        unsigned* bar; cudaMalloc(&bar, 256); cudaMemset(bar, 0, 256);
        void* args[] = {&bar, &cyc, nullptr}; int rounds = 200; args[2] = &rounds;
        cudaLaunchCooperativeKernel((void*)gridbar_kernel, dim3(sms), dim3(256), args, 0, 0); cudaDeviceSynchronize();
        printf("grid barrier (%d CTAs, red.release + ld.acquire poll): %lld cycles per barrier  [%s]\n", sms, cyc[0], cudaGetErrorString(cudaGetLastError()));
    }
    for (int kb : {16, 64}) {
        uint4* src; cudaMalloc(&src, kb * 1024); cudaMemset(src, 1, kb * 1024);
        uint4* sink; cudaMalloc(&sink, sms * 16);
        cudaFuncSetAttribute(bcast_read_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536);
        for (int rep = 0; rep < 2; ++rep) { bcast_read_kernel<<<sms, 256, 65536>>>(src, kb * 64, sink, cyc); cudaDeviceSynchronize(); }
        long long mx = 0, mn = 1ll << 60; for (int i = 0; i < sms; ++i) { if (cyc[i] > mx) mx = cyc[i]; if (cyc[i] < mn) mn = cyc[i]; }
        printf("all %d CTAs read the same %d KB into smem (256 thr): min %lld max %lld cycles\n", sms, kb, mn, mx);
        bcast_read_kernel<<<1, 256, 65536>>>(src, kb * 64, sink, cyc); cudaDeviceSynchronize();
        printf("   one CTA alone: %lld cycles\n", cyc[0]);
    }
    return 0;
}
