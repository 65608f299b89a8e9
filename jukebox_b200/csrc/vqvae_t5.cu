// ResConv1DBlock of the VQ-VAE decoder side on the Hopper tensor cores (wgmma), TMA-staged.
//
//   out = x + res_scale * (W2 . relu(W1 * relu(x) + b1) + b2)        (vqvae/resnet.py:27-44: k3 dilated conv, k1 conv)
//
// Channels-last fp32 [N, T, C] in and out, C in {32, 64}.  Same arithmetic as resblock_h2_kernel (vqvae_kernels.cu): every
// product runs as the split-precision triple  hi.w_hi + lo.w_hi + hi.w_lo  of fp16 halves (hi = fp16(v), lo = fp16(v - hi):
// 22 significant bits) accumulated in fp32 - but the MMAs are warpgroup MMAs (wgmma m64nCk16) reading both operands
// from swizzled shared memory, where mma.sync needs a ldmatrix per fragment and leaves the legacy tensor path saturated.
//
// One persistent CTA per SM walks tiles of 128 positions; three roles, connected by mbarriers only.  The tap pipeline
// below (tap_producer, tap_converter, tap_accumulate) is shared with conv_t5_kernel:
//   last warp   TMA producer   cp.async.bulk.tensor.3d of the fp32 rows of one tap, [128 rows x C] of clip n starting at
//                              t0 + (tap - 1) * dilation, into a ring.  Rows outside [0, T) arrive as zeros (the tensor
//                              map's out-of-bounds fill IS the convolution's zero padding).
//   warps 8..   converters     fp32 tap tile -> relu -> hi / lo fp16 planes in the K-major, 128-byte-swizzled layout the
//                              tensor core reads (row r, 16-byte chunk j at r * 128 + ((j ^ (r & 7)) << 4)), 2-stage ring
//   warps 0-7   consumers      two warpgroups, rows 0-63 and 64-127 of the tile: per tap C / 16 k-steps x 3 products into
//                              accumulator 1 (registers); then hidden = relu(acc / 2^8 + b1) split into hi / lo fp16
//                              pairs IN REGISTERS - the accumulator fragment is the A fragment of the next wgmma - and the
//                              k1 conv (hidden . W2) into accumulator 2; then x + res_scale * (acc / 2^8 + b2) through a
//                              shared-memory stage so that the residual loads and the stores are coalesced.
// W1 / W2 are scaled by 2^8 before the split (undone in the epilogues) so that their fp16 remainders stay out of the
// subnormal range; both are split and laid out (N-major rows, K contiguous, same swizzle) once per CTA.
#include "split_tma.cuh"
#include <algorithm>

using namespace jk;

namespace {

template <int C>
struct T5 {
    // converter groups of 4 warps (group g converts the taps whose counter is g mod 2): two for C = 32, one for C = 64
    // (C = 64 has no shared memory left for a deeper fp32 ring); + 8 consumer warps and the producer warp
    static constexpr int kGroups = C == 64 ? 1 : 2, kThreads = 32 * (9 + 4 * kGroups);
    static constexpr int kWBlock = C * 128;                 // one K block of a weight plane: C rows x 128 bytes
    static constexpr int kW1 = 3 * kWBlock, kW2 = kWBlock;   // bytes per plane
    static constexpr int kATile = kBM * 128;                 // one operand plane of a tap tile (128-byte rows)
    static constexpr int kFTile = kBM * C * 4;               // fp32 tap tile as TMA delivers it
    static constexpr int kFS = C == 64 ? 2 : 4;              // stages of the fp32 ring (what shared memory leaves room for)
    static constexpr int offW1h = 0, offW1l = kW1, offW2h = 2 * kW1, offW2l = 2 * kW1 + kW2;
    static constexpr int offA = 2 * kW1 + 2 * kW2;           // [2 stages][hi | lo]
    static constexpr int offS = offA + 2 * 2 * kATile;       // output stage [128][C] fp32
    static constexpr int offF = offS + kBM * C * 4;          // [kFS stages] fp32
    static constexpr int offBias = offF + kFS * kFTile;      // b1, b2
    static constexpr int offBar = offBias + 2 * C * 4;
    static constexpr int smem = offBar + 256;
};

// scale * (acc / 2^8 + bias) of one consumer warpgroup's 64 rows -> stage[row][C], 16-byte chunks XOR-swizzled with row & 7
template <int C>
__device__ __forceinline__ void stage_rows(float* stage, const float (&acc)[C / 2], const float* bias, float scale, int row0, int lane) {
#pragma unroll
    for (int j = 0; j < C / 4; ++j) {                     // j = 2 i + h: columns 8 i + 2 (lane % 4) + {0, 1}, row + 8 h
        const int row = row0 + 8 * (j & 1), col = 8 * (j >> 1) + 2 * (lane & 3);
        float2 o;
        o.x = scale * fmaf(acc[2 * j], kWInv, bias[col]);
        o.y = scale * fmaf(acc[2 * j + 1], kWInv, bias[col + 1]);
        *reinterpret_cast<float2*>(stage + row * C + (((col >> 2) ^ (row & 7)) << 2) + (col & 3)) = o;
    }
}

// ---- the tap pipeline -----------------------------------------------------------------
// Barriers at bars: f_full[4] | f_empty[4] (fp32 ring, FS of them used) | a_full[2] | a_empty[2] (operand slots).
template <int FS>
__device__ __forceinline__ void tap_init(uint64_t* bars, const CUtensorMap* map) {
    uint64_t *f_full = bars, *f_empty = bars + 4, *a_full = bars + 8, *a_empty = bars + 10;
    for (int i = 0; i < FS; ++i) { mbar_init(&f_full[i], 1); mbar_init(&f_empty[i], 128); }
    for (int i = 0; i < 2; ++i) { mbar_init(&a_full[i], 128); mbar_init(&a_empty[i], 2); }   // a_empty: one arrival per warpgroup
    mbar_fence_init();
    prefetch_tensormap(map);
}

// w[(tap * CI + ci) * CO + co] (n = taps * CI * CO values) -> 2^8 w split into the planes hi / lo [tap][row co][k ci]
template <int CI, int CO, int kThreads>
__device__ __forceinline__ void split_weight(const float* __restrict__ w, int n, uint8_t* hi, uint8_t* lo) {
    for (int i = threadIdx.x; i < n; i += kThreads) {
        const int tap = i / (CI * CO), ci = (i / CO) % CI, co = i % CO;
        __half h, l;
        split_f16(kWScale * __ldg(w + i), h, l);
        const uint32_t o = tap * (CO * 128) + sw_off(co, ci >> 3) + (ci & 7) * 2;
        *reinterpret_cast<__half*>(hi + o) = h;
        *reinterpret_cast<__half*>(lo + o) = l;
    }
}

// one lane: the fp32 rows of every tap of every tile this CTA takes, at row t0 + off(tap) of clip nb.  kPrefetch: the
// rows of the tiles this CTA takes next are pulled into L2 two iterations ahead
template <class L, bool kPrefetch, class Off>
__device__ __forceinline__ void tap_producer(const CUtensorMap* map, uint8_t* sm, uint64_t* bars, int ntap, Off off,
                                             int tiles_per_clip, int total_tiles) {
    constexpr int FS = L::kFS;
    uint64_t *f_full = bars, *f_empty = bars + 4;
    const int first = blockIdx.x, stride = gridDim.x;
    auto prefetch = [&](int tile) {
        if (tile >= total_tiles) return;
        const int nb = tile / tiles_per_clip, t0 = (tile - nb * tiles_per_clip) * kBM;
        for (int tap = 0; tap < ntap; ++tap)
            asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(
                             reinterpret_cast<uint64_t>(map)), "r"(0), "r"(t0 + off(tap)), "r"(nb) : "memory");
    };
    if constexpr (kPrefetch) prefetch(first + stride);
    uint32_t kt = 0;
    for (int tile = first; tile < total_tiles; tile += stride) {
        const int nb = tile / tiles_per_clip, t0 = (tile - nb * tiles_per_clip) * kBM;
        if constexpr (kPrefetch) prefetch(tile + 2 * stride);
        for (int tap = 0; tap < ntap; ++tap, ++kt) {
            const int s = kt % FS;
            mbar_wait(&f_empty[s], ((kt / FS) & 1) ^ 1);
            mbar_expect_tx(&f_full[s], (uint32_t)L::kFTile);
            tma_load_3d(sm + L::offF + s * L::kFTile, map, 0, t0 + off(tap), nb, &f_full[s]);
        }
    }
}

// fp32 tap tiles -> (relu) -> hi / lo planes of the operand slots, by kGroups groups of 128 threads (warps 8..).  With two
// groups, group g takes the taps whose counter is g mod 2 - that is the operand slot g and the fp32 slots g (mod 2) - so
// two taps are converted concurrently and every barrier still sees exactly the 128 arrivals of one group per use
template <class L, int C, int kGroups>
__device__ __forceinline__ void tap_converter(uint8_t* sm, uint64_t* bars, int ntap, bool relu, int total_tiles) {
    constexpr int FS = L::kFS;
    uint64_t *f_full = bars, *f_empty = bars + 4, *a_full = bars + 8, *a_empty = bars + 10;
    const int cg = ((threadIdx.x >> 5) - 8) >> 2, ct = threadIdx.x & 127;
    uint32_t kt = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        for (int tap = 0; tap < ntap; ++tap, ++kt) {
            if (kGroups == 2 && (int)(kt & 1) != cg) continue;
            const int s = kt & 1, fs = kt % FS;
            mbar_wait(&f_full[fs], (kt / FS) & 1);
            mbar_wait(&a_empty[s], ((kt >> 1) & 1) ^ 1);
            convert_planes<C / 4, false, false>(sm + L::offF + fs * L::kFTile, sm + L::offA + s * 2 * L::kATile, ct, relu);
            // The fp32 slot is released only here, after every loaded value has been consumed by the stores above (an
            // arrive right behind the loads would let TMA refill the slot under them); the proxy fence also orders this
            // thread's generic reads of the slot before the async-proxy writes of the refill.
            fence_async_smem();
            mbar_arrive(&a_full[s]);
            mbar_arrive(&f_empty[fs]);
        }
    }
}

// one consumer warpgroup's rows of one tile: acc = sum over the taps of A(tap) . W(tap) (planes wh / wl, one K block per
// tap); each tap's operand slot is freed as soon as wgmma.wait_group 1 says it retired
template <class L, int CI, int CO>
__device__ __forceinline__ void tap_accumulate(float (&acc)[CO / 2], uint32_t& kt, int ntap, uint8_t* sm, uint64_t* bars,
                                               int wg, int wt, uint32_t wh, uint32_t wl) {
    uint64_t *a_full = bars + 8, *a_empty = bars + 10;
#pragma unroll
    for (int i = 0; i < CO / 2; ++i) acc[i] = 0.f;
    for (int tap = 0; tap < ntap; ++tap, ++kt) {
        const int s = kt & 1;
        mbar_wait(&a_full[s], (kt >> 1) & 1);
        const uint32_t ah = smem_u32(sm + L::offA + s * 2 * L::kATile) + wg * (64 * 128), al = ah + L::kATile;
        mma_tap<CI, CO>(acc, ah, al, wh + tap * L::kWBlock, wl + tap * L::kWBlock);
        if (tap > 0) {                                // the previous tap has retired: free its operand slot
            wgmma_wait<1>();
            if (wt == 0) mbar_arrive(&a_empty[(kt - 1) & 1]);
        }
    }
    wgmma_wait<0>();
    if (wt == 0) mbar_arrive(&a_empty[(kt - 1) & 1]);
}

template <int C>
__global__ void __launch_bounds__(T5<C>::kThreads, 1)
resblock_t5_kernel(const __grid_constant__ CUtensorMap map_x, const float* __restrict__ x, float* __restrict__ out,
                   const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                   const float* __restrict__ b2, long long T, int dil, float rs, int tiles_per_clip, int total_tiles) {
    using L = T5<C>;
    constexpr int kGroups = L::kGroups, kThreadsT5 = L::kThreads, kProducer = 8 + 4 * kGroups;
    extern __shared__ __align__(1024) uint8_t sm[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + L::offBar);
    float* bias = reinterpret_cast<float*>(sm + L::offBias);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    // ---- once per CTA: barriers, weights (scaled, split, swizzled), biases ------------------------------------------
    if (tid == 0) tap_init<L::kFS>(bars, &map_x);
    split_weight<C, C, kThreadsT5>(w1, 3 * C * C, sm + L::offW1h, sm + L::offW1l);
    split_weight<C, C, kThreadsT5>(w2, C * C, sm + L::offW2h, sm + L::offW2l);
    for (int i = tid; i < 2 * C; i += kThreadsT5) bias[i] = i < C ? __ldg(b1 + i) : __ldg(b2 + i - C);
    fence_async_smem();                                       // the weight planes are read by the tensor core (async proxy)
    __syncthreads();
    const int first = blockIdx.x, stride = gridDim.x;

    if (warp == kProducer) {
        // every row is read three times, as the centre tap of one tile and the side taps of two others: whoever comes first
        // pays the HBM latency, so the L2 prefetch makes the ring's loads L2 hits - a ring of 64 KB cannot cover an HBM
        // round trip
        if (lane == 0)
            tap_producer<L, true>(&map_x, sm, bars, 3, [dil](int tap) { return (tap - 1) * dil; }, tiles_per_clip, total_tiles);
    } else if (warp >= 8) {
        tap_converter<L, C, kGroups>(sm, bars, 3, true, total_tiles);
    } else {
        // ================= consumers: conv1, hidden tile, conv2, output =================
        const int wg = warp >> 2, wt = tid & 127, row0 = wg * 64 + (wt >> 5) * 16 + (lane >> 2);
        const uint32_t w1h = smem_u32(sm + L::offW1h), w1l = smem_u32(sm + L::offW1l);
        const uint32_t w2h = smem_u32(sm + L::offW2h), w2l = smem_u32(sm + L::offW2l);
        float* stage = reinterpret_cast<float*>(sm + L::offS);
        constexpr int CH4 = C / 4;
        uint32_t kt = 0;
        for (int tile = first; tile < total_tiles; tile += stride) {
            const int nb = tile / tiles_per_clip, t0 = (tile - nb * tiles_per_clip) * kBM;
            float acc[C / 2];
            tap_accumulate<L, C, C>(acc, kt, 3, sm, bars, wg, wt, w1h, w1l);
            // ---- hidden = relu(conv1 / 2^8 + b1) -> hi / lo A fragments of the k1 conv -------------------------------
            uint32_t hh[C / 16][4], hl[C / 16][4];
#pragma unroll
            for (int j = 0; j < C / 4; ++j) {                 // j = 2 i + h: register 2 (i & 1) + h of k-step i / 2
                const int col = 8 * (j >> 1) + 2 * (lane & 3);
                const float a0 = fmaxf(fmaf(acc[2 * j], kWInv, bias[col]), 0.f);
                const float a1 = fmaxf(fmaf(acc[2 * j + 1], kWInv, bias[col + 1]), 0.f);
                split_f16x2(a0, a1, hh[j >> 2][j & 3], hl[j >> 2][j & 3]);
            }
            // this thread's share of the residual rows of its warpgroup (coalesced), requested while the k1 conv runs
            const float* xin = x + ((size_t)nb * T + t0) * C;
            float4 xres[CH4 / 2];
#pragma unroll
            for (int i = 0; i < CH4 / 2; ++i) {
                const int item = wg * 64 * CH4 + wt + i * 128;
                xres[i] = ((long long)t0 + item / CH4 < T) ? __ldg(reinterpret_cast<const float4*>(xin) + item) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            // ---- k1 conv: hidden . W2 -------------------------------------------------------------------------------
#pragma unroll
            for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < C / 16; ++k) {
                wgmma_rs<C>(acc, hl[k], wgmma_desc_sw128(w2h + k * 32));
                wgmma_rs<C>(acc, hh[k], wgmma_desc_sw128(w2l + k * 32));
                wgmma_rs<C>(acc, hh[k], wgmma_desc_sw128(w2h + k * 32));
            }
            wgmma_commit();
            wgmma_wait<0>();
            // ---- out = x + res_scale * (conv2 / 2^8 + b2) -----------------------------------------------------------
            // a thread holds pieces of two rows; the tile goes through shared memory so that the residual loads and the
            // stores run with consecutive lanes on consecutive 16-byte chunks
            stage_rows<C>(stage, acc, bias + C, rs, row0, lane);
            named_sync(1 + wg);
            {
                float* xo = out + ((size_t)nb * T + t0) * C;
#pragma unroll
                for (int i = 0; i < CH4 / 2; ++i) {
                    const int item = wg * 64 * CH4 + wt + i * 128, rr = item / CH4, jj = item % CH4;
                    if ((long long)t0 + rr < T) {
                        const float4 v = *reinterpret_cast<const float4*>(stage + rr * C + ((jj ^ (rr & 7)) << 2));
                        const float4 xr = xres[i];
                        *(reinterpret_cast<float4*>(xo) + item) = make_float4(v.x + xr.x, v.y + xr.y, v.z + xr.z, v.w + xr.w);
                    }
                }
            }
            named_sync(1 + wg);                                // the stage rows are rewritten by the next tile
        }
    }
}

// ---------------------------------------------------------------------------------------
// Tap-GEMM convolution on the same tap pipeline, for the decoder-side convs BETWEEN the residual blocks (the k3 input conv
// of a DecoderConvBock, the two 2-tap phases of its k4-s2 transposed convs; encdec.py:28-46):
//   out[t * os + oo, :] = res + scale * (sum_j x[t + off_j, :] . W_j + b),   c_in, c_out in {32, 64}, <= 3 taps, stride-1 input.
// Roles as in resblock_t5_kernel minus the hidden tile: two consumer warpgroups (warps 0-7) that accumulate in registers
// and stage scale * (acc / 2^8 + b) through shared memory to add the residual / store whole rows coalesced, 4 converter
// warps (8-11), one TMA producer warp (12).
// ---------------------------------------------------------------------------------------
struct ConvT5P {
    const float* in; float* out; const float* w; const float* bias; const float* res;
    long long t_in, t_out;
    int n_taps, tap_off[3], out_stride, out_offset, relu_in;
    float scale;
};

template <int CI, int CO>
struct T5C {
    static constexpr int kWBlock = CO * 128;                 // one tap of a weight plane: CO rows x 128 bytes (K = CI <= 64)
    static constexpr int kW = 3 * kWBlock;                   // bytes per plane (<= 3 taps)
    static constexpr int kATile = kBM * 128;
    static constexpr int kFTile = kBM * CI * 4;
    static constexpr int kFS = CI == 64 ? 2 : 4;
    static constexpr int offWh = 0, offWl = kW;
    static constexpr int offA = 2 * kW;                      // [2 stages][hi | lo]
    static constexpr int offS = offA + 2 * 2 * kATile;       // output staging [128][CO] fp32
    static constexpr int offF = offS + kBM * CO * 4;
    static constexpr int offBias = offF + kFS * kFTile;
    static constexpr int offBar = offBias + CO * 4;
    static constexpr int smem = offBar + 256;
};
constexpr int kConvThreads = 416;

template <int CI, int CO>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_t5_kernel(const __grid_constant__ CUtensorMap map_x, ConvT5P P, int tiles_per_clip, int total_tiles) {
    using L = T5C<CI, CO>;
    extern __shared__ __align__(1024) uint8_t sm[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(sm + L::offBar);
    float* bias = reinterpret_cast<float*>(sm + L::offBias);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ntap = P.n_taps;
    if (tid == 0) tap_init<L::kFS>(bars, &map_x);
    split_weight<CI, CO, kConvThreads>(P.w, ntap * CI * CO, sm + L::offWh, sm + L::offWl);
    for (int i = tid; i < CO; i += kConvThreads) bias[i] = P.bias ? __ldg(P.bias + i) : 0.f;
    fence_async_smem();
    __syncthreads();
    const int first = blockIdx.x, stride = gridDim.x;

    if (warp == 12) {
        if (lane == 0) {
            auto off = [&](int tap) { return tap == 0 ? P.tap_off[0] : tap == 1 ? P.tap_off[1] : P.tap_off[2]; };   // no local copy of the array
            tap_producer<L, false>(&map_x, sm, bars, ntap, off, tiles_per_clip, total_tiles);
        }
    } else if (warp >= 8) {
        tap_converter<L, CI, 1>(sm, bars, ntap, P.relu_in != 0, total_tiles);
    } else {
        const int wg = warp >> 2, wt = tid & 127, row0 = wg * 64 + (wt >> 5) * 16 + (lane >> 2);
        const uint32_t wh = smem_u32(sm + L::offWh), wl = smem_u32(sm + L::offWl);
        float* stage = reinterpret_cast<float*>(sm + L::offS);
        const long long rows_out = P.t_out * P.out_stride;
        uint32_t kt = 0;
        for (int tile = first; tile < total_tiles; tile += stride) {
            const int nb = tile / tiles_per_clip, t0 = (tile - nb * tiles_per_clip) * kBM;
            float acc[CO / 2];
            tap_accumulate<L, CI, CO>(acc, kt, ntap, sm, bars, wg, wt, wh, wl);
            stage_rows<CO>(stage, acc, bias, P.scale, row0, lane);
            named_sync(1 + wg);
            {
                constexpr int CH4 = CO / 4;
                float* ob = P.out + (size_t)nb * rows_out * CO;
                const float* rb = P.res ? P.res + (size_t)nb * rows_out * CO : nullptr;
#pragma unroll 4
                for (int i = 0; i < CH4 / 2; ++i) {
                    const int item = wg * 64 * CH4 + wt + i * 128, rr = item / CH4, jj = item % CH4;
                    const long long t = (long long)t0 + rr;
                    if (t < P.t_out) {
                        float4 v = *reinterpret_cast<const float4*>(stage + rr * CO + ((jj ^ (rr & 7)) << 2));
                        const size_t o = (size_t)(t * P.out_stride + P.out_offset) * CO + jj * 4;
                        if (rb) {
                            const float4 xr = __ldg(reinterpret_cast<const float4*>(rb + o));
                            v.x += xr.x; v.y += xr.y; v.z += xr.z; v.w += xr.w;
                        }
                        *reinterpret_cast<float4*>(ob + o) = v;
                    }
                }
            }
            named_sync(1 + wg);
        }
    }
}

// ---------------------------------------------------------------------------------------
// Wide tap-GEMM convolution on the streamed-weight pipeline (split_tma.cuh), for c_in, c_out multiples of 64 with one of
// them above 64 (the upsampler Conditioner's 512 / 1024 / 1920 channels, prior/conditioners.py):
//   out[t * os + oo, co0 .. co0 + BN) = res + scale * (sum_tap sum_ci x[t + off_tap, ci] . W[tap, ci, co] + b)
// K = taps x c_in no longer fits one operand tile and the weights no longer fit in shared memory, so
//   - a work item is 128 positions x BN output channels (BN = 128, or 64 when c_out is an odd multiple of 64).  Items are
//     numbered position-tile major: the CTAs that work on the channel tiles of one position tile at the same time share
//     its activation rows in L2;
//   - the K loop runs over the 64-channel blocks of every tap.  A stage's weight planes come straight from the split
//     weight that jk_pack_conv_weight_split made once per weight load ([hi | lo][c_out][taps * c_in] fp16 of 2^8 w);
//   - the epilogue writes scale * (acc / 2^8 + b) (+ res) from the accumulator fragments: the four lanes of a quad cover
//     32 contiguous bytes of one row (whole sectors, also for the row-strided phases of a transposed conv), and shared
//     memory is left to the ring.
// ---------------------------------------------------------------------------------------
struct ConvWideP {
    const float* bias; const float* res; float* out;
    long long t_out;
    int c_in, c_out, n_taps, tap_off[3], out_stride, out_offset, relu_in;
    float scale;
};

template <int BN>
struct ConvWideJob {
    using Ring = StreamRing<BN, BN == 128 ? 3 : 4>;          // ring stages: what 227 KB of shared memory leaves room for
    static constexpr bool kCheck = false;
    const CUtensorMap *map_a, *map_w;                        // [c_in, t_in, n] fp32 activations, the split weight
    ConvWideP P;
    int tiles_per_clip, n_tiles_n, kb_per_tap, n_kb;
    bool relu;
    struct Tile { int nb, t0, co0; };

    __device__ __forceinline__ Tile tile(int item) const {
        const int mt = item / n_tiles_n, co0 = (item - mt * n_tiles_n) * BN;
        const int nb = mt / tiles_per_clip, t0 = (mt - nb * tiles_per_clip) * kBM;
        return {nb, t0, co0};
    }
    __device__ __forceinline__ void load(uint8_t* st, const Tile& t, int kb, uint64_t* bar) const {
        const int tap = kb / kb_per_tap, c0 = (kb - tap * kb_per_tap) * 64;
        const int off = tap == 0 ? P.tap_off[0] : tap == 1 ? P.tap_off[1] : P.tap_off[2];
        // rows outside [0, T) of clip nb - a whole block of them when the dilation exceeds T - arrive as zeros
        tma_load_3d(st, map_a, c0, t.t0 + off, t.nb, bar);
        tma_load_2d(st + Ring::kA, map_w, tap * P.c_in + c0, t.co0, bar);
        tma_load_2d(st + Ring::kA + Ring::kB, map_w, tap * P.c_in + c0, P.c_out + t.co0, bar);
    }
    // ---- out = res + scale * (acc / 2^8 + b), straight from the fragments ----
    __device__ __forceinline__ void epilogue(const float (&acc)[BN / 2], const Tile& t, int rq, int lane) const {
        const long long rows_out = P.t_out * P.out_stride;
        float* ob = P.out + (size_t)t.nb * rows_out * P.c_out + t.co0;
        const float* rb = P.res ? P.res + (size_t)t.nb * rows_out * P.c_out + t.co0 : nullptr;
        const float* bb = P.bias ? P.bias + t.co0 : nullptr;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const long long tt = (long long)t.t0 + rq + 8 * h;
            if (tt < P.t_out) {
                const size_t ro = (size_t)(tt * P.out_stride + P.out_offset) * P.c_out;
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    const int col = 8 * i + 2 * (lane & 3);
                    const float2 b = bb ? __ldg(reinterpret_cast<const float2*>(bb + col)) : make_float2(0.f, 0.f);
                    float2 o;
                    o.x = P.scale * fmaf(acc[4 * i + 2 * h], kWInv, b.x);
                    o.y = P.scale * fmaf(acc[4 * i + 2 * h + 1], kWInv, b.y);
                    if (rb) {
                        const float2 r = __ldg(reinterpret_cast<const float2*>(rb + ro + col));
                        o.x += r.x; o.y += r.y;
                    }
                    *reinterpret_cast<float2*>(ob + ro + col) = o;
                }
            }
        }
    }
};

template <int BN>
__global__ void __launch_bounds__(kStreamThreads, 1)
conv_wide_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, ConvWideP P,
                 int tiles_per_clip, int n_tiles_n, int total_items) {
    extern __shared__ __align__(1024) uint8_t sm_raw[];
    const int kb_per_tap = P.c_in / 64;
    const ConvWideJob<BN> job{&map_x, &map_w, P, tiles_per_clip, n_tiles_n, kb_per_tap, P.n_taps * kb_per_tap, P.relu_in != 0};
    streamed_pipeline(job, sm_raw, total_items);
}

// packed fp32 [k, c_in, c_out] -> [hi | lo][c_out][k * c_in] fp16 of 2^8 w (row co, column tap * c_in + ci)
__global__ void pack_split_kernel(const float* __restrict__ packed, unsigned short* __restrict__ split, int K, int c_out) {
    const long long total = (long long)K * c_out;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int kk = (int)(i / c_out), co = (int)(i % c_out);   // coalesced reads of the packed weight
        __half h, l;
        split_f16(kWScale * __ldg(packed + i), h, l);
        const size_t o = (size_t)co * K + kk;
        split[o] = __half_as_ushort(h);
        split[(size_t)K * c_out + o] = __half_as_ushort(l);
    }
}

template <int C>
int launch_t5(const float* x, float* out, const float* w1, const float* b1, const float* w2, const float* b2, int n,
              long long T, int dil, float rs, cudaStream_t stream) {
    CUtensorMap map;
    if (int rc = encode_rows_map(&map, x, n, T, C, C)) return rc;
    int sms = 0;
    if (int rc = set_max_smem_once<resblock_t5_kernel<C>>(T5<C>::smem)) return rc;
    if (int rc = sm_count(&sms)) return rc;
    const long long per_clip = (T + kBM - 1) / kBM, total = per_clip * n;
    JK_REQUIRE(total < (1ll << 31) && T + 4096 < (1ll << 31), "clip too long for 32-bit tile coordinates");
    const unsigned grid = (unsigned)std::min<long long>(total, sms);
    resblock_t5_kernel<C><<<grid, T5<C>::kThreads, T5<C>::smem, stream>>>(map, x, out, w1, b1, w2, b2, T, dil, rs, (int)per_clip, (int)total);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}


template <int CI, int CO>
int launch_conv_t5(const ConvT5P& P, int n, cudaStream_t stream) {
    CUtensorMap map;
    if (int rc = encode_rows_map(&map, P.in, n, P.t_in, CI, CI)) return rc;
    int sms = 0;
    if (int rc = set_max_smem_once<conv_t5_kernel<CI, CO>>(T5C<CI, CO>::smem)) return rc;
    if (int rc = sm_count(&sms)) return rc;
    const long long per_clip = (P.t_out + kBM - 1) / kBM, total = per_clip * n;
    JK_REQUIRE(total < (1ll << 31) && P.t_in + 4096 < (1ll << 31), "clip too long for 32-bit tile coordinates");
    const unsigned grid = (unsigned)std::min<long long>(total, sms);
    conv_t5_kernel<CI, CO><<<grid, kConvThreads, T5C<CI, CO>::smem, stream>>>(map, P, (int)per_clip, (int)total);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <int BN>
int launch_conv_wide(const float* in, long long t_in, const void* w_split, const ConvWideP& P, int n, cudaStream_t stream) {
    constexpr int kSmem = ConvWideJob<BN>::Ring::smem;
    CUtensorMap map_x, map_w;
    if (int rc = encode_rows_map(&map_x, in, n, t_in, P.c_in, 64)) return rc;
    const long long K = (long long)P.n_taps * P.c_in;
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)2 * P.c_out};
    const cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)BN};
    if (int rc = encode_tensor_map(&map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w_split, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
        return rc;
    int sms = 0;
    if (int rc = set_max_smem_once<conv_wide_kernel<BN>>(kSmem)) return rc;
    if (int rc = sm_count(&sms)) return rc;
    const long long per_clip = (P.t_out + kBM - 1) / kBM, n_tiles_n = P.c_out / BN, total = per_clip * n * n_tiles_n;
    JK_REQUIRE(total < (1ll << 31) && t_in + 4096 < (1ll << 31), "clip too long for 32-bit tile coordinates");
    const unsigned grid = (unsigned)std::min<long long>(total, sms);
    conv_wide_kernel<BN><<<grid, kStreamThreads, kSmem, stream>>>(map_x, map_w, P, (int)per_clip, (int)n_tiles_n, (int)total);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}
}  // namespace

namespace jk {
// vqvae_kernels.cu (jk_resblock_tc) dispatches here when the shape qualifies: C in {32, 64}, T >= 128, 16-byte aligned
int resblock_t5(const float* x, float* out, const float* w1, const float* b1, const float* w2, const float* b2, int n,
                long long T, int C, int dil, float rs, cudaStream_t stream) {
    if (C == 64) return launch_t5<64>(x, out, w1, b1, w2, b2, n, T, dil, rs, stream);
    if (C == 32) return launch_t5<32>(x, out, w1, b1, w2, b2, n, T, dil, rs, stream);
    JK_REQUIRE(false, "resblock_t5: C must be 32 or 64 (got %d)", C);
    return 0;
}
// jk_conv1d_cl with tensor_cores = 1 dispatches here: stride-1 input, <= 3 taps, c_in / c_out in {32, 64}, t_in >= 128
int conv_t5(const float* in, long long t_in, int c_in, float* out, long long t_out, int c_out, const float* w, const float* bias,
            const float* res, int n_taps, const int* tap_off, int out_stride, int out_offset, int relu_in, float scale, int n,
            cudaStream_t stream) {
    ConvT5P P;
    P.in = in; P.out = out; P.w = w; P.bias = bias; P.res = res; P.t_in = t_in; P.t_out = t_out; P.n_taps = n_taps;
    for (int i = 0; i < 3; ++i) P.tap_off[i] = i < n_taps ? tap_off[i] : 0;
    P.out_stride = out_stride; P.out_offset = out_offset; P.relu_in = relu_in; P.scale = scale;
    if (c_in == 64 && c_out == 64) return launch_conv_t5<64, 64>(P, n, stream);
    if (c_in == 64 && c_out == 32) return launch_conv_t5<64, 32>(P, n, stream);
    if (c_in == 32 && c_out == 64) return launch_conv_t5<32, 64>(P, n, stream);
    if (c_in == 32 && c_out == 32) return launch_conv_t5<32, 32>(P, n, stream);
    JK_REQUIRE(false, "conv_t5: channels must be 32 or 64 (got %d -> %d)", c_in, c_out);
    return 0;
}
// jk_conv1d_tc_wide (vqvae_kernels.cu) dispatches here once it has checked the shape: c_in, c_out multiples of 64,
// stride-1 input, <= 3 taps, t_in >= 128, 16-byte aligned pointers; w_split from pack_conv_weight_split
int conv_wide_t5(const float* in, long long t_in, int c_in, float* out, long long t_out, int c_out, const void* w_split,
                 const float* bias, const float* res, int n_taps, const int* tap_off, int out_stride, int out_offset,
                 int relu_in, float scale, int n, cudaStream_t stream) {
    ConvWideP P;
    P.bias = bias; P.res = res; P.out = out; P.t_out = t_out; P.c_in = c_in; P.c_out = c_out; P.n_taps = n_taps;
    for (int i = 0; i < 3; ++i) P.tap_off[i] = i < n_taps ? tap_off[i] : 0;
    P.out_stride = out_stride; P.out_offset = out_offset; P.relu_in = relu_in; P.scale = scale;
    if (c_out % 128 == 0) return launch_conv_wide<128>(in, t_in, w_split, P, n, stream);
    return launch_conv_wide<64>(in, t_in, w_split, P, n, stream);
}
int pack_conv_weight_split(const float* packed, void* split, int k, int c_in, int c_out, cudaStream_t stream) {
    const long long total = (long long)k * c_in * c_out;
    const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, 65535);
    pack_split_kernel<<<blocks, 256, 0, stream>>>(packed, static_cast<unsigned short*>(split), k * c_in, c_out);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}
}  // namespace jk
