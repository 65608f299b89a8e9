// Persistent decode-step engine for Jukebox's autoregressive priors on H100 (sm_90a).
//
// One launch = one token position for up to 32 samples through the WHOLE transformer stack
// (reference: ConditionalAutoregressive2D.sample loop body, prior/autoregressive.py:222-237,
//  -> Transformer.forward(sample=True), transformer/transformer.py:169-192).
//
// Why this shape (DESIGN.md has the numbers).  At n_samples <= 16 the step is HBM-bound on weight streaming
// (83-99 % of the bytes) but a 72-layer stack is a chain of 360 dependent phases, each needing what EVERY SM
// produced in the previous one.  Round 1 paid a grid-wide barrier (1.2-1.7 us) plus a 148-fold redundant
// activation staging (1-2 us) per phase and sat at 0.14 of the HBM roofline.  This version has NO grid barrier:
//   * grid = #SMs persistent CTAs (cooperative launch: co-residency), 8 consumer warps + 1 producer warp
//   * weights are pre-packed (jk_prior_load_layer) into one contiguous byte stream per CTA, in consumption
//     order, in mma.sync B-fragment order.  The producer warp walks it with 1-D TMA bulk copies
//     (cp.async.bulk -> SASS UBLKCP) into a shared-memory ring guarded by full/empty mbarriers and runs ahead
//     of the compute phases by the ring's depth.
//   * CTAs are grouped in units of KS (4 for 1b_lyrics): a unit owns 8-column groups of every Conv1D, its KS
//     CTAs split K.  So a CTA stages only K/KS of the activations (and LayerNorms only that), runs
//     [16 x K/KS] x [K/KS x 8*ncg] on mma.sync m16n8k16, and the KS partial sums meet through an exchange
//     buffer; each CTA then finishes 1/KS of the unit's columns (bias, quick_gelu / residual, fp16 rounding).
//   * every producer -> consumer hand-over is an "LL" exchange (NCCL's low-latency protocol): a value travels
//     as one 8-byte word {data, flag} written by a single store; the consumer polls the word itself.  One
//     L2 round trip instead of release-counter + acquire-poll + data load, and arrival skew is absorbed word
//     by word.  Flags are unique per (step, layer), nothing is ever reset.
//   * LayerNorm statistics need all columns of a row: producers add sum / sum-of-squares of their columns
//     into 64-bit fixed-point words (exact, order independent) whose top bits count the contributing CTAs;
//     the LN consumers poll the words until the count says every CTA has added.  These two all-to-all points
//     per layer are also what makes buffer reuse safe (see "hazards" below).
//   * the residual stream never leaves the SM: the CTA that finishes columns c of proj finishes the same
//     columns of proj2 (and of the embedding), so h / x1 slices live in shared memory.
//   * KV caches are laid out per attention pattern so that the rows a token attends are one contiguous run
//     (transpose-block layers store position p at row (p % bc)*blocks + p / bc).
//
// Hazards.  A buffer written once per layer may be overwritten for layer l+1 only after every reader of layer
// l is done.  Every writer first passes an LN statistics wait of layer l+1 (a statistics word all G CTAs add to
// AFTER their previous phases, in program order), so all reads of layer l happen-before it.
// The partial-sum exchange has one buffer per Conv1D index for the same reason.
//
// Numerics: activations fp16, accumulation fp32, LayerNorm/softmax fp32 - see oracle/transformer_np.py.
#include "engine.cuh"
#include <cooperative_groups.h>
#include <vector>
#include <algorithm>
#include <string.h>
#include <stdlib.h>
#include <math.h>

using namespace jk;

namespace {

constexpr int kConsumers = 256;
constexpr int kThreads = 384;          // 2 consumer warpgroups (8 warps) + 1 producer warpgroup (warp 8 works, 9-11 exit)
constexpr int kSlotBytes = 16384;
constexpr int kMaxSlots = 12;
constexpr int kHeaderBytes = 8192;     // barriers, LN statistics, descriptor / layer records, residual slice
constexpr int kLogitKT = 1024;         // K tile (floats) of the fp32 logits product at 16 rows
constexpr int kLogitRowsPerChunk = 4;
constexpr int kLogitRowsPerPass = 16;
constexpr int kMaxSplit = 4;
constexpr int kProfSlots = 1024;
constexpr int kXpCols = 64;            // columns per unit in the partial-sum exchange (8 groups of 8)
// The decode kernel is instantiated for R = 16 and R = 32 activation rows (the M of the MMAs: one or two m16 tiles
// against every weight fragment); jk_prior_step launches the 16-row kernel whenever n_samples <= 16.
// cross-warp reduction tile [8 warps][R rows][<= 72 floats]
__host__ __device__ constexpr int red_bytes(int R) { return 8 * R * 72 * 4; }
// K tile of the fp32 logits product: its y tile [R][kt] floats stays at 64 KB
__host__ __device__ constexpr int logit_kt(int R) { return kLogitKT * 16 / R; }
// LayerNorm statistics words: [63:52] number of CTAs that have contributed, [51:0] fixed-point value
constexpr int kCntShift = 52;
constexpr unsigned long long kValMask = (1ull << kCntShift) - 1;
constexpr long long kSumBias = 1ll << 41;      // per contribution, keeps the sum field non-negative

struct StepArgs {
    int n;
    const float* x_in;
    const long long* tokens;
    long long tok_stride;
    const float* y_cond;
    const float* x_cond;
    long long x_cond_len;
    float* h_out;
    float* logits;
    long long logits_bstride, logits_tstride;
    const float* logit_bias;            // x_cond . x_out^T per position (jkb200.h), or NULL
    long long lb_bstride, lb_tstride;
};

// per-launch record of the logits GEMM in the shared-memory header (written by the kernel before each pass)
struct LogitsRec {
    float* lg_out;              // logits of this position
    long long lg_bs;
    const float* lb;            // logit bias of this position or NULL
    long long lb_bs;
    unsigned long long* xp;     // partial-sum exchange of the current pass: xp[pass]
    ushort2 cols;               // column groups of this unit in the current pass
};
// values of a launch in the shared-memory header (written once by the kernel prologue, see launch_pos())
struct LaunchVals {
    int pm, pd;                 // p % block_ctx, p / block_ctx
    int gmax;                   // CTAs available per (sample, head)
    int t;                      // position p
    unsigned step;              // steps executed before this launch
};
// thread layout of the activation staging for one K (see stage_map_init)
struct StageDim {
    int cw, rgc;
};

// The one dynamic shared-memory block of the decode kernel.  Every device function derives its
// pointers from this symbol (never from pointer parameters): that is what lets the compiler emit
// LDS/STS/ATOMS instead of generic LD/ST (measured: generic loads of the B fragments made the MMA loop
// 6x slower than the tensor pipe allows).
extern __shared__ __align__(1024) uint8_t jk_smem[];

// Its header [0, kHeaderBytes): byte offset and size of every region, in address order.  Only the accessors below
// address the header.
constexpr int kHdrBar = 0, kHdrBarBytes = 2 * kMaxSlots * 8;           // ring mbarriers: full[kMaxSlots], empty[kMaxSlots]
constexpr int kHdrStats = 256, kHdrStatsBytes = 32 * 2 * 4;            // LayerNorm statistics [R rows] {-mean * rstd, rstd}
constexpr int kHdrDesc = 512, kHdrDescBytes = 512;                     // descriptor head: EngineDev up to `layer`
constexpr int kHdrLayer = 1024, kHdrLayerSlot = 256;                   // two layer slots (layer l in slot l & 1): LayerDev,
constexpr int kHdrColsAt = 128;                                        //   and at +kHdrColsAt this unit's ushort2 cols[4]
constexpr int kHdrRes = 2048, kHdrResBytes = 16 * 32 * 8;              // residual-stream slice of this CTA, see res_ld()
static_assert(kHdrResBytes == 32 * 32 * 4, "the 32-row residual slice (half2) must fill the 16-row one (float2)");
constexpr int kHdrMap = 6144, kHdrMapBytes = 3 * kConsumers * 2;       // staging thread layouts [3 kinds][kConsumers]
constexpr int kHdrMapDim = 7680, kHdrMapDimBytes = 3 * (int)sizeof(StageDim);
constexpr int kHdrLaunch = 7712, kHdrLaunchBytes = (int)sizeof(LaunchVals);
constexpr int kHdrLrec = 7744, kHdrLrecBytes = (int)sizeof(LogitsRec);
static_assert(offsetof(EngineDev, layer) <= kHdrDescBytes, "descriptor head must fit its shared-memory slot");
static_assert(sizeof(LayerDev) <= kHdrColsAt && kHdrColsAt + 4 * sizeof(ushort2) <= kHdrLayerSlot,
              "layer record and column assignment must fit their shared-memory slot");
static_assert(kHdrBar + kHdrBarBytes <= kHdrStats && kHdrStats + kHdrStatsBytes <= kHdrDesc &&
              kHdrDesc + kHdrDescBytes <= kHdrLayer && kHdrLayer + 2 * kHdrLayerSlot <= kHdrRes &&
              kHdrRes + kHdrResBytes <= kHdrMap && kHdrMap + kHdrMapBytes <= kHdrMapDim &&
              kHdrMapDim + kHdrMapDimBytes <= kHdrLaunch && kHdrLaunch + kHdrLaunchBytes <= kHdrLrec &&
              kHdrLrec + kHdrLrecBytes <= kHeaderBytes,
              "shared-memory header regions overlap or exceed kHeaderBytes");

__device__ __forceinline__ uint64_t* sm_full() { return reinterpret_cast<uint64_t*>(jk_smem + kHdrBar); }
__device__ __forceinline__ uint64_t* sm_empty() { return sm_full() + kMaxSlots; }
__device__ __forceinline__ float* sm_stats() { return reinterpret_cast<float*>(jk_smem + kHdrStats); }
// Entry i = row * 32 + column pair of this CTA's residual-stream slice: [16][32] float2 at 16 rows, [32][32] half2 at
// 32 rows.  Every value stored is already fp16-rounded, so the half form is exact and the slice keeps its 4 KB.
template <int R>
__device__ __forceinline__ float2 res_ld(int i) {
    if constexpr (R == 16) return reinterpret_cast<const float2*>(jk_smem + kHdrRes)[i];
    else return __half22float2(reinterpret_cast<const __half2*>(jk_smem + kHdrRes)[i]);
}
template <int R>
__device__ __forceinline__ void res_st(int i, float2 v) {
    if constexpr (R == 16) reinterpret_cast<float2*>(jk_smem + kHdrRes)[i] = v;
    else reinterpret_cast<__half2*>(jk_smem + kHdrRes)[i] = __floats2half2_rn(v.x, v.y);
}
__device__ __forceinline__ uint8_t* sm_uni() { return jk_smem + kHeaderBytes; }
// The engine descriptor lives in global memory; with the shared-memory carve-out at its maximum there is
// no L1 to cache it, so every `E->field` was an L2 round trip (~300 cycles) on the dependency chain.
// The head of the descriptor (everything before the per-layer array) and the current / next layer
// records are therefore copied into shared memory once and read with LDS.
__device__ __forceinline__ uint32_t* sm_desc_words() { return reinterpret_cast<uint32_t*>(jk_smem + kHdrDesc); }
__device__ __forceinline__ const EngineDev* sm_E() { return reinterpret_cast<const EngineDev*>(jk_smem + kHdrDesc); }
__device__ __forceinline__ uint8_t* sm_layer_slot(int l) { return jk_smem + kHdrLayer + kHdrLayerSlot * (l & 1); }
__device__ __forceinline__ const LayerDev* sm_layer(int l) { return reinterpret_cast<const LayerDev*>(sm_layer_slot(l)); }
// (first 8-column group, number of groups) of this unit in layer l's QKV, proj, fc and proj2
__device__ __forceinline__ ushort2* sm_cols(int l) { return reinterpret_cast<ushort2*>(sm_layer_slot(l) + kHdrColsAt); }
__device__ __forceinline__ unsigned short* sm_stage_map(int kind) {
    return reinterpret_cast<unsigned short*>(jk_smem + kHdrMap + 2 * kConsumers * kind);
}
__device__ __forceinline__ StageDim* sm_stage_dim(int kind) { return reinterpret_cast<StageDim*>(jk_smem + kHdrMapDim) + kind; }
__device__ __forceinline__ LaunchVals* sm_launch() { return reinterpret_cast<LaunchVals*>(jk_smem + kHdrLaunch); }
__device__ __forceinline__ LogitsRec* sm_lrec() { return reinterpret_cast<LogitsRec*>(jk_smem + kHdrLrec); }

// Position in the weight ring.  Only the slot and its parity travel (in registers) through the phase calls; the slot
// count and slot 0's offset are per-launch constants read from the descriptor in shared memory where they are needed, so
// that ptxas' inter-procedural allocation has two registers more for the phase functions.
struct Ring {
    int slot;
    uint32_t phase;
    __device__ __forceinline__ static int nslot() { return sm_E()->nslot; }
    __device__ __forceinline__ uint64_t* full() const { return sm_full() + slot; }
    __device__ __forceinline__ uint64_t* empty() const { return sm_empty() + slot; }
    __device__ __forceinline__ uint8_t* data() const {
        const EngineDev* E = sm_E();
        return jk_smem + kHeaderBytes + E->uni_bytes + E->kvpre_bytes + slot * kSlotBytes;
    }
    __device__ __forceinline__ void advance() {
        if (++slot == nslot()) { slot = 0; phase ^= 1u; }
    }
};

#define STAMP(E_, slot_, i_)                                                                \
    do {                                                                                    \
        if (blockIdx.x == 0 && threadIdx.x == 0 && (E_)->prof_on && (slot_) < kProfSlots)      \
            (E_)->prof2[(size_t)(slot_) * 8 + (i_)] = clock64();                             \
    } while (0)

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// k-steps per ring slot for a unit of ncg column groups: the largest power of two with k * ncg * 256 B <= 16 KB
__device__ __host__ __forceinline__ int kpc_of(int ncg) { return ncg == 1 ? 64 : ncg == 2 ? 32 : ncg <= 4 ? 16 : 8; }

// ---- LL words ------------------------------------------------------------------------------
// 8 bytes = {data (low 32 bits), flag (high 32 bits)}.  A naturally aligned 8-byte access is single-copy
// atomic, so a reader that sees the flag sees the data; relaxed gpu-scope accesses go to L2 (no L1).
#define JK_ST_LL "st.relaxed.gpu.global"
__device__ __forceinline__ void ll_st(unsigned long long* p, uint32_t data, uint32_t flag) {
    const unsigned long long v = ((unsigned long long)flag << 32) | data;
    asm volatile(JK_ST_LL ".u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Polled loads are relaxed gpu-scope loads (SASS LDG.E.STRONG.GPU).  A weak ld.global.cg compiles to the SAME SASS load
// on sm_90a, but ptxas may hoist a weak load out of the polling loop (it did: the weak build deadlocked into the spin
// guard), so the strong form is the only usable one.
__device__ __forceinline__ ulonglong2 ll_ld2(const unsigned long long* p) {
    ulonglong2 v;
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ll_ld1(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// tuning aid (JK_NOWAIT=1): hand-overs stop waiting (results are garbage) - what remains is every CTA's own work, so
// step time with and without it separates "waiting for other SMs" from "work on the critical path of one SM"
__constant__ int jk_nowait;
__device__ __forceinline__ bool ll_ok(unsigned long long w, uint32_t flag) { return ((uint32_t)(w >> 32) == flag) | (jk_nowait != 0); }
__device__ __forceinline__ void spin_guard(unsigned& spins) {
    if (++spins > (1u << 24)) __trap();     // a protocol bug traps instead of hanging the GPU
}
// a statistics word whose count field says every CTA has contributed
__device__ __forceinline__ unsigned long long wait_stat_word(const long long* p, int G) {
    unsigned spins = 0;
    unsigned long long w = ll_ld1(reinterpret_cast<const unsigned long long*>(p));
    while ((int)(w >> kCntShift) != G && !jk_nowait) { spin_guard(spins); w = ll_ld1(reinterpret_cast<const unsigned long long*>(p)); }
    return w;
}

// quick_gelu(x) = x * sigmoid(1.702 x) (transformer/ops.py:33-35).  The reference's eager fp16 path
// rounds after each of its three elementwise ops; restated exactly so (x is already an fp16 value).
__device__ __forceinline__ float quick_gelu_f(float x) {
    const float z = h2f_round(1.702f * x);
    const float s = h2f_round(1.0f / (1.0f + expf(-z)));
    return x * s;
}

// ---------------------------------------------------------------------------------------
// LayerNorm statistics travel with the activations: whoever WRITES columns of the residual stream also adds
// sum(x) and sum(x^2) of its columns into per-row 64-bit fixed-point accumulators (integer adds => order
// independent => bit-reproducible), so the consuming GEMM can normalise while it stages - no extra pass over
// the row.  The SAME word counts contributors in its top 12 bits: every CTA adds exactly once per LayerNorm
// (CTAs without columns add an empty contribution), so "count == G" means the value is complete and the
// consumer simply polls the word - one red and one poll, no separate counter, no fence.
//   sum  : x rounded to 2^-16 per element (a pure function of x), biased by 2^41 per contribution
//   sumsq: min(x^2, 2^24) rounded to 2^-14 per element
// Worst case (8192 columns at the fp16 maximum) stays below 2^52, so the count field cannot be corrupted.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ long long fx_sum(float x) { return __float2ll_rn(x * 65536.0f); }
__device__ __forceinline__ long long fx_sq(float x) { return __float2ll_rn(fminf(x * x, 16777216.0f) * 16384.0f); }
__device__ __forceinline__ void red_add_u64(long long* p, unsigned long long v) {
    atomicAdd(reinterpret_cast<unsigned long long*>(p), v);
}
template <int R>
__device__ __forceinline__ long long* sm_sfx() { return reinterpret_cast<long long*>(sm_uni() + red_bytes(R)); }

// This CTA's contribution to the statistics block `ln_out` ([32 rows] x {sum, sumsq} adjacent, one 128-byte line per row).
// sfx: [2][32 rows][32] fixed-point values of the column pairs it wrote.  32 threads each
// reduce one (row, moment) in a fixed order and issue ONE 64-bit red carrying value + count.
template <int R>
__device__ __forceinline__ void publish_stats(long long* ln_out, int B, int ppc) {
    const int tid = threadIdx.x;
    consumer_sync();
    if (tid < 2 * B) {
        const long long* sfx = sm_sfx<R>() + (tid & 1) * 1024;
        const int row = tid >> 1;
        long long s = (tid & 1) ? 0 : kSumBias;
        for (int i = 0; i < ppc; ++i) s += sfx[row * 32 + i];
        red_add_u64(ln_out + 16 * row + (tid & 1), (1ull << kCntShift) + (unsigned long long)s);
    }
    consumer_sync();                       // the scratch is reused by the next phase
}

// activation staging: LL words of rows [0, B), columns [k0, k0 + Ks) -> shared fp16 [R][Ks+8] (ldmatrix
// friendly), optionally through LayerNorm (fp32 math, eps 1e-5; reference transformer/ops.py:14-24).
// Threads are laid out [row group][8-column vector]: a thread keeps ONE column vector (gamma / beta loaded
// once) and walks rows rg, rg + rgc, ...; four rows = eight 16-byte polled loads in flight per batch.
// Rows >= B are never written: an MMA output row depends only on its own A row, and those outputs are discarded.
// How the 256 consumer threads tile a [R rows][Ks / 8 vectors] slice: cw column vectors per pass x rgc row groups,
// thread -> (column vector cv, row group rg).  Computed once per launch for the three K of a layer (kind 0: width,
// 1: n_state, 2: mlp width) and kept in the shared-memory header: sm_stage_map(kind)[tid] = cv | rg << 8,
// sm_stage_dim(kind) = {cw, rgc} - so no integer division sits on the path of a phase.
__device__ __forceinline__ void stage_map_init(int kind, int Ks) {
    const int nvec = Ks >> 3, tid = threadIdx.x;
    const int cw = nvec >= kConsumers ? kConsumers : nvec;
    const int rgc = nvec >= kConsumers ? 1 : kConsumers / nvec;
    sm_stage_map(kind)[tid] = (unsigned short)((tid % cw) | ((tid / cw) << 8));
    if (tid == 0) {
        sm_stage_dim(kind)->cw = cw;
        sm_stage_dim(kind)->rgc = rgc;
    }
}

template <int R>
__device__ __forceinline__ void stage_acts_body(const unsigned long long* in, int K, int k0, int Ks, int B, uint32_t flag, int ln,
                                                const float* gamma, const float* beta, const long long* lnacc, int kind, int pslot) {
    const int tid = threadIdx.x;
    uint8_t* acts = sm_uni();
    float* stats = sm_stats();
    const int nvec = Ks >> 3;
    const int astride = (Ks + 8) * 2;
    // LayerNorm statistics of the R rows: thread r polls the two adjacent words (sum, sum of squares) of row r with one
    // 16-byte load until every CTA has contributed to both (R pollers per CTA on R lines).  Called AFTER this thread's
    // activation loads are issued: on the R polling threads the two latencies overlap instead of adding up.
    auto row_statistics = [&]() {
        const int G = sm_E()->G;
        float mean = 0.f, rstd = 0.f;
        if (tid < B) {
            const unsigned long long* wp = reinterpret_cast<const unsigned long long*>(lnacc + 16 * tid);
            unsigned spins = 0;
            ulonglong2 w = ll_ld2(wp);
            while (((int)(w.x >> kCntShift) != G || (int)(w.y >> kCntShift) != G) && !jk_nowait) { spin_guard(spins); w = ll_ld2(wp); }
            const long long val = (long long)(w.x & kValMask) - (long long)G * kSumBias, sq = (long long)(w.y & kValMask);
            // double only for the cancellation in E[x^2] - mean^2 (adds / muls; no double div or sqrt:
            // those are kilobytes of library code in the instruction cache)
            const double rk = (double)(1.0f / (float)K);    // K is a multiple of 16: exact for powers of two, 1e-7 rel otherwise
            const double m = (double)val * (1.0 / 65536.0) * rk;
            double var = fma(rk, (double)sq * (1.0 / 16384.0), -(m * m));   // one rounding: oracle/decode_stats.py states it so
            var = var < 0.0 ? 0.0 : var;
            rstd = 1.0f / sqrtf((float)var + 1e-5f);
            mean = -(float)m * rstd;                        // staged as x * rstd + (-mean * rstd), then * gamma + beta
        }
        stats[2 * tid] = mean;
        stats[2 * tid + 1] = rstd;
        STAMP(sm_E(), pslot, 5);
    };
    const int cw = sm_stage_dim(kind)->cw, rgc = sm_stage_dim(kind)->rgc;
    const unsigned tm = sm_stage_map(kind)[tid];
    const int cv = tm & 255, rg = tm >> 8;
    const int row_words = K >> 1;
    bool stats_ready = !ln;
#pragma unroll 1
    for (int vb = 0; vb < nvec; vb += cw) {
        const int v = vb + cv;
        const bool act = (v < nvec) && (rg < rgc);
        float gm[8], bt[8];
        if (act && ln) {      // issued first: their latency overlaps the polled loads below
            *reinterpret_cast<float4*>(gm) = __ldg(reinterpret_cast<const float4*>(gamma + k0 + v * 8));
            *reinterpret_cast<float4*>(gm + 4) = __ldg(reinterpret_cast<const float4*>(gamma + k0 + v * 8 + 4));
            *reinterpret_cast<float4*>(bt) = __ldg(reinterpret_cast<const float4*>(beta + k0 + v * 8));
            *reinterpret_cast<float4*>(bt + 4) = __ldg(reinterpret_cast<const float4*>(beta + k0 + v * 8 + 4));
        }
#pragma unroll 1
        for (int r0 = rg; r0 < R; r0 += 4 * rgc) {           // uniform trip count per thread group: barrier below
            ulonglong2 w[4][2];
            auto issue = [&]() {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int r = r0 + j * rgc;
                    if (r < B) {
                        const unsigned long long* src = in + (size_t)r * row_words + ((k0 + v * 8) >> 1);
                        w[j][0] = ll_ld2(src);
                        w[j][1] = ll_ld2(src + 2);
                    }
                }
            };
            if (act) issue();
            if (!stats_ready && tid < R) row_statistics();       // (ln only) while the loads above are in flight
            if (act) {
                unsigned spins = 0;
                for (;;) {
                    bool again = false;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int r = r0 + j * rgc;
                        if (r < B)
                            again |= !(ll_ok(w[j][0].x, flag) && ll_ok(w[j][0].y, flag) && ll_ok(w[j][1].x, flag) &&
                                       ll_ok(w[j][1].y, flag));
                    }
                    if (!again) break;
                    spin_guard(spins);
                    issue();
                }
            }
            STAMP(sm_E(), pslot, 6);                                        // this thread's polled loads are in
            if (!stats_ready) { consumer_sync(); stats_ready = true; }     // row statistics are in shared memory
            STAMP(sm_E(), pslot, 7);
            if (act) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int r = r0 + j * rgc;
                    if (r < B) {
                        uint4 x = make_uint4((uint32_t)w[j][0].x, (uint32_t)w[j][0].y, (uint32_t)w[j][1].x, (uint32_t)w[j][1].y);
                        if (ln) {
                            __half2* hp = reinterpret_cast<__half2*>(&x);
                            const float rstd = stats[2 * r + 1], nmr = stats[2 * r];     // nmr = -mean * rstd
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                float2 f = __half22float2(hp[e]);
                                f.x = fmaf(fmaf(f.x, rstd, nmr), gm[2 * e], bt[2 * e]);
                                f.y = fmaf(fmaf(f.y, rstd, nmr), gm[2 * e + 1], bt[2 * e + 1]);
                                hp[e] = __floats2half2_rn(f.x, f.y);
                            }
                        }
                        *reinterpret_cast<uint4*>(acts + r * astride + v * 16) = x;
                    }
                }
            }
        }
    }
    if (!stats_ready) { if (tid < R) row_statistics(); consumer_sync(); }
}
// The 16-row GEMM phase calls the staging as a function of its own; the 32-row one inlines it.  Called at 32 rows, the
// staging left gemm_phase too few registers for what it keeps across the call: ptxas put one word (the return address)
// in local memory, an L2 round trip per phase.  Without the call the staging's registers and the two accumulator sets
// are simply disjoint live ranges.
template <int R>
__device__ __noinline__ void stage_acts(const unsigned long long* in, int K, int k0, int Ks, int B, uint32_t flag, int ln,
                                        const float* gamma, const float* beta, const long long* lnacc, int kind, int pslot) {
    stage_acts_body<R>(in, K, k0, Ks, B, flag, ln, gamma, beta, lnacc, kind, pslot);
}

__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// nk k-steps of one ring slot, by one warp: its k-steps x column groups are independent MMAs that pipeline back to
// back.  NCG (8-column groups of this unit) is a template parameter: with a run-time count the compiler serialised
// every LDS -> HMMA pair through one register pair (tools/micro/ubench.cu: 4070 vs 1170 cycles for the K = 2048 loop).
// MT m16 row tiles (R = 16 * MT rows; tile m starts at arow + m * atile): each B fragment is loaded from the ring slot
// once and multiplied into MT accumulator sets.  With two tiles one k-step already issues 2 * NCG independent MMAs, and
// the loop stays rolled: unrolled by 2 it made gemm_phase<32> spill (STL 1 / LDL 2, and STL 11 in the kernel body).
template <int NCG, int MT>
__device__ __forceinline__ void mma_chunk(float (&acc)[MT][8][4], uint32_t arow, uint32_t atile, uint32_t sl, int kk0, int nk) {
#pragma unroll (MT == 1 ? 4 : 1)
    for (int i = 0; i < nk; ++i) {
        uint32_t a[MT][4];
#pragma unroll
        for (int m = 0; m < MT; ++m) ldsm4(a[m], arow + m * atile + (kk0 + i) * 32);
        uint2 b[NCG];
#pragma unroll
        for (int j = 0; j < NCG; ++j) b[j] = lds64(sl + ((i * NCG + j) << 8));
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int j = 0; j < NCG; ++j) mma_16816(acc[m][j], a[m], b[j].x, b[j].y);
    }
}

// ---------------------------------------------------------------------------------------
// one Conv1D at decode.  Unit u owns columns [8*g0, 8*(g0+ncg)); this CTA (rank r of the unit) owns the K slice
// [r*K/KS, (r+1)*K/KS):  partial[R, 8*ncg] = acts[R, K/KS] . Wslice, exchanged inside the unit, and this CTA
// finishes column pairs [r*ppc, (r+1)*ppc) of the unit: out = epilogue(sum of the KS partials in rank order).
// ---------------------------------------------------------------------------------------
enum { EPI_QKV = 0, EPI_PROJ = 1, EPI_FC = 2, EPI_PROJ2 = 3, EPI_LOGITS = 4 };

struct GemmArgs {
    const unsigned long long* in;       // LL input [rows][K/2]
    unsigned long long* out;            // LL output [rows][N/2]
    unsigned long long* xp;             // partial-sum exchange of this Conv1D index
    int K, N, g0, ncg, ln, epi, pslot;
    uint32_t flag_in, flag_out;
    const float *gamma, *beta, *bias;
    const long long* ln_in;             // statistics block behind the input (LayerNorm phases)
    long long* ln_out;                  // statistics block of the rows this epilogue writes (residual epilogues)
    int kind;                           // 0: K = width, 1: K = n_state, 2: K = mlp width (thread layout of the staging)
    int kin;                            // columns of one LL input row (= K, except the logits GEMM: K = 2 * kin)
    float* lg_out;                      // EPI_LOGITS: fp32 logits of this position, row stride lg_bs
    long long lg_bs;
    const float* lb;                    // EPI_LOGITS: logit bias of this position (or NULL), row stride lb_bs
    long long lb_bs;
};

// One Conv1D of layer l (or the logits GEMM), identified by its epilogue.  The argument record is assembled HERE from the
// descriptor / layer record / column table in shared memory: passed by value it had grown past what the call ABI keeps in
// registers (896 bytes of stack), and with the shared-memory carve-out at its maximum every local-memory access is an L2
// round trip - the step went from 1.95 to 2.5 ms.
template <int R>
__device__ __noinline__ Ring gemm_phase(Ring ring, int B, int epi_, int l, int pslot_, uint32_t fl) {
    const EngineDev* E = sm_E();
    GemmArgs g;
    {
        const LayerDev& LD = *sm_layer(l);
        const ushort2* cl = sm_cols(l);
        const int W = E->W, S = E->S, M = E->M;
        long long* lnb = E->lnacc + (size_t)(2 * l) * 512;
        g.epi = epi_; g.pslot = pslot_; g.flag_in = fl; g.flag_out = fl;
        g.gamma = nullptr; g.beta = nullptr; g.ln_in = nullptr; g.ln_out = nullptr; g.ln = 0;
        g.lg_out = nullptr; g.lg_bs = 0; g.lb = nullptr; g.lb_bs = 0;
        if (epi_ == EPI_QKV) {
            g.in = E->ll_h; g.out = E->ll_qkv; g.xp = E->xp[0]; g.K = W; g.N = (LD.attn_func == 6) ? S : 3 * S;
            g.g0 = cl[0].x; g.ncg = cl[0].y; g.ln = 1; g.gamma = LD.ln0_g; g.beta = LD.ln0_b; g.bias = LD.b_qkv;
            g.ln_in = lnb; g.kind = 0; g.kin = W;
        } else if (epi_ == EPI_PROJ) {
            g.in = E->ll_a; g.out = E->ll_x1; g.xp = E->xp[1]; g.K = S; g.N = W; g.g0 = cl[1].x; g.ncg = cl[1].y;
            g.bias = LD.b_o; g.ln_out = lnb + 512; g.kind = 1; g.kin = S;
        } else if (epi_ == EPI_FC) {
            g.in = E->ll_x1; g.out = E->ll_g; g.xp = E->xp[2]; g.K = W; g.N = M; g.g0 = cl[2].x; g.ncg = cl[2].y;
            g.ln = 1; g.gamma = LD.ln1_g; g.beta = LD.ln1_b; g.bias = LD.b_1; g.ln_in = lnb + 512; g.kind = 0; g.kin = W;
        } else if (epi_ == EPI_PROJ2) {
            g.in = E->ll_g; g.out = E->ll_h; g.xp = E->xp[3]; g.K = M; g.N = W; g.g0 = cl[3].x; g.ncg = cl[3].y;
            g.bias = LD.b_2; g.ln_out = lnb + 1024; g.flag_out = fl + 1; g.kind = 2; g.kin = M;
        } else {       // EPI_LOGITS: [y | y] x [hi(x_out) ; lo(x_out)], see the kernel
            const LogitsRec* lr = sm_lrec();
            g.in = E->ll_h; g.out = nullptr; g.xp = lr->xp; g.K = 2 * W; g.N = E->bins; g.g0 = lr->cols.x; g.ncg = lr->cols.y;
            g.bias = nullptr; g.kind = 2; g.kin = W; g.flag_out = 0;
            g.lg_out = lr->lg_out; g.lg_bs = lr->lg_bs; g.lb = lr->lb; g.lb_bs = lr->lb_bs;
        }
    }
    uint8_t* uni = sm_uni();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int KS = E->KS, ksh = E->ks_shift, c = blockIdx.x, rank = c & (KS - 1);
    const int ncg = g.ncg, nc = ncg * 8;
    const int ppc = (nc >> 1) >> ksh;                    // column pairs this CTA finishes
    const bool residual = (g.epi == EPI_PROJ || g.epi == EPI_PROJ2);
    STAMP(E, g.pslot, 0);
    if (ncg == 0) {                                      // a unit without columns (tiny models) still contributes (count only)
        if (residual) publish_stats<R>(g.ln_out, B, 0);
        return ring;
    }
    const int K = g.K, N = g.N, epi = g.epi;
    const int Ks = K >> ksh;
    // the logits GEMM multiplies [y | y] with [hi(x_out) ; lo(x_out)]: its K runs twice over the kin input columns
    const int k0 = rank * Ks - (rank * Ks >= g.kin ? g.kin : 0);
    if constexpr (R == 16) stage_acts<R>(g.in, g.kin, k0, Ks, B, g.flag_in, g.ln, g.gamma, g.beta, g.ln_in, g.kind, g.pslot);
    else stage_acts_body<R>(g.in, g.kin, k0, Ks, B, g.flag_in, g.ln, g.gamma, g.beta, g.ln_in, g.kind, g.pslot);
    consumer_sync();
    STAMP(E, g.pslot, 1);

    constexpr int MT = R / 16;                            // m16 row tiles
    float acc[MT][8][4];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int j = 0; j < 8; ++j) { acc[m][j][0] = acc[m][j][1] = acc[m][j][2] = acc[m][j][3] = 0.f; }
    const int nkk = Ks >> 4;
    const int kpc = kpc_of(ncg);                          // a power of two
    const int astride = (Ks + 8) * 2;
    const uint32_t arow = smem_u32(uni + (lane & 15) * astride + (lane >> 4) * 16);
    const uint32_t atile = 16 * astride;
    // The k-steps of this CTA's slice are dealt to the eight warps in contiguous runs (k-step i -> warp i * 8 / nkk), so
    // every warp multiplies - 4 k-steps each for a K = 2048 / KS = 4 phase instead of four warps with a whole slot each and
    // four idle.  EVERY warp still waits for every slot and arrives on its empty barrier, in order: the parity protocol of
    // the ring only holds while no warp is a whole ring ahead of or behind the producer.
    int k_lo, k_hi;
    if (nkk >= 8) { k_lo = (warp * nkk) >> 3; k_hi = ((warp + 1) * nkk) >> 3; }
    else { k_lo = min(warp, nkk); k_hi = min(warp + 1, nkk); }
    // A warp waits only for the slots it multiplies from when the whole phase fits the ring (a slot index then occurs at
    // most once per phase, and the CTA barriers between phases keep the warps within one phase of each other, so an early
    // arrival on a foreign slot's empty barrier always belongs to the barrier's current pass); a phase longer than the ring
    // (5b_lyrics: 38 slots, 6 in the ring) keeps every warp in the producer's order.  An already-complete try_wait costs
    // ~90 cycles: three of them per warp per phase were pure overhead.
    // In such a long phase the slots go round robin to the warps instead (slot s -> warp s mod 8, the whole slot): with
    // contiguous runs one warp would own several consecutive slots while the ring delivers them in order, i.e. one warp
    // would multiply at a time (5b_lyrics, one box: 6 192 us per step round robin, 6 691 us with contiguous runs).
    const int nslots_phase = (nkk + kpc - 1) >> (31 - __clz(kpc));
    const bool in_order = nslots_phase > Ring::nslot();
    int slot_i = 0;
#define JK_MMA_LOOP(NCG)                                                                      \
    {                                                                                         \
        _Pragma("unroll 1") for (int kk0 = 0; kk0 < nkk; kk0 += kpc, ++slot_i) {              \
            int a_ = max(kk0, k_lo), b_ = min(min(kk0 + kpc, nkk), k_hi);                     \
            if (in_order) { a_ = kk0; b_ = ((slot_i & 7) == warp) ? min(kk0 + kpc, nkk) : kk0; } \
            if (a_ < b_ || in_order) mbar_wait(ring.full(), ring.phase);                       \
            if (a_ < b_)                                                                      \
                mma_chunk<NCG, MT>(acc, arow, atile, smem_u32(ring.data()) + lane * 8 + (((a_ - kk0) * NCG) << 8), a_, b_ - a_); \
            __syncwarp();                                                                      \
            if (lane == 0) mbar_arrive(ring.empty());                                          \
            ring.advance();                                                                   \
        }                                                                                     \
    }
    switch (ncg) {
        case 1: JK_MMA_LOOP(1) break;
        case 2: JK_MMA_LOOP(2) break;
        case 3: JK_MMA_LOOP(3) break;
        case 4: JK_MMA_LOOP(4) break;
        case 5: JK_MMA_LOOP(5) break;
        case 6: JK_MMA_LOOP(6) break;
        case 7: JK_MMA_LOOP(7) break;
        default: JK_MMA_LOOP(8) break;
    }
#undef JK_MMA_LOOP
    STAMP(E, g.pslot, 2);
    const int nwarp = in_order ? min(8, nslots_phase) : min(8, nkk);       // warps that multiplied at least one k-step
    float* red = reinterpret_cast<float*>(uni);
    const int ncp = ((nc + 31) & ~31) + 8;
    // partial sums of the unit: [KS ranks][R rows][64 columns] LL words {fp32, flag}
    unsigned long long* xp_unit = g.xp + (size_t)(c - rank) * R * kXpCols;
    {
        consumer_sync();                   // everyone is done reading the staged activations
        // cross-warp reduction tile [warps that owned a slot][R rows][ncp floats]; ncp = 8 mod 32 keeps both the fragment
        // stores below and the row-wise pair loads of the epilogue free of bank conflicts
        if (warp < nwarp) {
            const int r0 = lane >> 2, c0 = (lane & 3) * 2;
#pragma unroll
            for (int m = 0; m < MT; ++m) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (j < ncg) {
                        float* d = red + (size_t)(warp * R + m * 16) * ncp + j * 8 + c0;
                        *reinterpret_cast<float2*>(d + r0 * ncp) = make_float2(acc[m][j][0], acc[m][j][1]);
                        *reinterpret_cast<float2*>(d + (r0 + 8) * ncp) = make_float2(acc[m][j][2], acc[m][j][3]);
                    }
                }
            }
        }
        consumer_sync();
        if (KS > 1 && lane < (nc >> 1)) {
            // one partial per rank: the warps' tiles summed here, published in slot 0 of this rank (lane = column pair,
            // warp = sample row and row + 8)
#pragma unroll 1
            for (int b = warp; b < B; b += 8) {
                float s0 = 0.f, s1 = 0.f;
                for (int w = 0; w < nwarp; ++w) {
                    const float2 v = *reinterpret_cast<const float2*>(red + (size_t)(w * R + b) * ncp + 2 * lane);
                    s0 += v.x; s1 += v.y;
                }
                unsigned long long* dst = xp_unit + ((size_t)rank * R + b) * kXpCols + 2 * lane;
                const unsigned long long fl = (unsigned long long)g.flag_in << 32;
                asm volatile(JK_ST_LL ".v2.u64 [%0], {%1,%2};" ::"l"(dst), "l"(fl | __float_as_uint(s0)),
                             "l"(fl | __float_as_uint(s1)) : "memory");
            }
        }
    }
    STAMP(E, g.pslot, 3);
    // ---- ... and finishes its own column pairs ----------------------------------------------------------
    long long* sfx = sm_sfx<R>();                                     // [2][32][32] statistics of the pairs written
    // thread layout: up to 16 pairs per CTA (every K-split configuration): half-warp = sample row (2 * warp + half, + 16),
    // lane & 15 = column pair; more pairs (KS = 1): lane = pair, rows warp, warp + 8, ...
    const bool two_rows = ppc <= 16;
    const int pl = two_rows ? (lane & 15) : lane;
    const int b_first = two_rows ? 2 * warp + (lane >> 4) : warp, b_step = two_rows ? 16 : 8;
    if (pl < ppc) {
        const int pr = rank * ppc + pl;                 // pair inside the unit
        const int gc = g.g0 * 8 + 2 * pr;               // global column of the pair
        const float2 bias = g.bias ? *reinterpret_cast<const float2*>(g.bias + gc) : make_float2(0.f, 0.f);
#pragma unroll 1
        for (int b = b_first; b < B; b += b_step) {
            float s0 = 0.f, s1 = 0.f;
            if (KS == 1) {
                for (int w = 0; w < nwarp; ++w) {
                    const float2 v = *reinterpret_cast<const float2*>(red + (size_t)(w * R + b) * ncp + 2 * pr);
                    s0 += v.x; s1 += v.y;
                }
            } else {
                // the KS partial words of this pair and row, polled together and summed in rank order: a fixed order, so
                // the result is bit-reproducible
                ulonglong2 v[4];
                unsigned spins = 0;
                bool again;
                do {
                    again = false;
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        if (q < KS) v[q] = ll_ld2(xp_unit + ((size_t)q * R + b) * kXpCols + 2 * pr);
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        if (q < KS) again |= !(ll_ok(v[q].x, g.flag_in) && ll_ok(v[q].y, g.flag_in));
                    if (again) spin_guard(spins);
                } while (again);
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (q < KS) { s0 += __uint_as_float((uint32_t)v[q].x); s1 += __uint_as_float((uint32_t)v[q].y); }
            }
            if (epi == EPI_LOGITS) {
                float* lo_ = g.lg_out + (size_t)b * g.lg_bs + gc;
                const float* lb_ = g.lb ? g.lb + (size_t)b * g.lb_bs + gc : nullptr;
                if (gc < N) lo_[0] = s0 + (lb_ ? lb_[0] : 0.f);
                if (gc + 1 < N) lo_[1] = s1 + (lb_ ? lb_[1] : 0.f);
                continue;
            }
            const float y0 = h2f_round(s0 + bias.x), y1 = h2f_round(s1 + bias.y);     // Conv1D output, rounded once to fp16
            __half2 o;
            if (epi == EPI_QKV) {
                o = __floats2half2_rn(y0, y1);
            } else if (epi == EPI_FC) {                        // quick_gelu (transformer/ops.py:33-35)
                o = __floats2half2_rn(quick_gelu_f(y0), quick_gelu_f(y1));
            } else {
                // EPI_PROJ : x1 = fp16(h + a)      EPI_PROJ2 : h = fp16(x1 + m)   (transformer.py:82-83)
                const float2 base = res_ld<R>(b * 32 + pl);
                const float o0 = h2f_round(base.x + y0), o1 = h2f_round(base.y + y1);
                res_st<R>(b * 32 + pl, make_float2(o0, o1));
                o = __floats2half2_rn(o0, o1);
                sfx[b * 32 + pl] = fx_sum(o0) + fx_sum(o1);
                sfx[1024 + b * 32 + pl] = fx_sq(o0) + fx_sq(o1);
            }
            ll_st(g.out + (size_t)b * (N >> 1) + (gc >> 1), *reinterpret_cast<const uint32_t*>(&o), g.flag_out);
        }
    }
    STAMP(E, g.pslot, 4);
    if (residual) publish_stats<R>(g.ln_out, B, ppc);
    else consumer_sync();                  // red region is reused by the next phase
    return ring;
}

// ---------------------------------------------------------------------------------------
// attention for one (sample, head, kv-split) work item; q_len == 1
// (reference: factored_attention.py:82-133 + per-pattern sample branches :135-228)
// ---------------------------------------------------------------------------------------
struct AttnGeom {
    int R;        // rows attended
    int base;     // first cache row of the attended run
    int cur;      // 1 if the current token is the last attended row
    int wrow;     // cache row the current token's k/v is written to (-1: none)
};

// pm = p % block_ctx, pd = p / block_ctx: computed once per launch
__device__ __forceinline__ AttnGeom attn_geom(const EngineDev* E, const LayerDev& LD, int p, int pm, int pd) {
    AttnGeom g;
    const int bc = E->bc;
    switch (LD.attn_func) {
        case 0: g.R = p + 1; g.base = 0; g.cur = 1; g.wrow = p; break;
        case 1: g.R = pm + 1; g.base = 0; g.cur = 1; g.wrow = pm; break;
        case 2: g.base = pm * E->blocks; g.R = pd + 1; g.cur = 1; g.wrow = g.base + pd; break;
        case 3:
            g.R = (p >= bc) ? bc : 0; g.base = ((pd + 1) & 1) * bc; g.cur = 0;
            g.wrow = (pd & 1) * bc + pm; break;
        case 7:
            g.R = min(p + 1, E->prime_pad); g.base = 0; g.cur = (p < E->prime_pad) ? 1 : 0;
            g.wrow = (p < E->prime_pad) ? p : -1; break;
        default: g.R = E->enc_dims; g.base = 0; g.cur = 0; g.wrow = -1; break;   // 6
    }
    return g;
}

// rows of one shared-memory K (or V) tile: a multiple of 16 (the MMA row block), ~24 KB per tile
__device__ __host__ __forceinline__ int attn_tile_rows(int dhp) {
    int r = (12288 / dhp) & ~15;
    return r < 16 ? 16 : (r > 64 ? 64 : r);
}

// how many CTAs share one (sample, head): as few as keep every part inside ONE shared-memory tile
// (RC - 1 cached rows + the current token's row), bounded by the grid
// (gmax = G / (B * H) is computed once per launch; no division here)
__device__ __forceinline__ int attn_nsplit(const EngineDev* E, int gmax, int ncache) {
    const int cap = E->RC - 1;
    const int ns = 1 + (ncache > cap) + (ncache > 2 * cap) + (ncache > 3 * cap);        // <= kMaxSplit
    return max(1, min(ns, gmax));
}
// x / d for d in 1..4 and 0 <= x < 98304
__device__ __forceinline__ int div_small(int x, int d) {
    return d == 1 ? x : d == 2 ? (x >> 1) : d == 4 ? (x >> 2) : (int)(((unsigned)x * 43691u) >> 17);
}

__device__ __forceinline__ void ldsm4_trans(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

// K/V tiles in shared memory: row r = dhp halves, its 16-byte chunks XOR-swizzled with (r & 7) so that
// ldmatrix (8 rows, same chunk) touches 8 different bank groups.  Only when a row has a multiple of 8
// chunks; other head sizes stay linear (correct, bank-conflicted).
__device__ __forceinline__ uint32_t kv_chunk_off(int r, int chunk, int dhp, int swz) {
    return (uint32_t)(r * dhp * 2 + ((chunk ^ (r & swz)) << 4));
}

// cp.async of rows [0, nr) of K and V into swizzled tiles.  Thread -> (first row, chunk) is fixed, so the
// loop body is two cp.async and two adds: no per-chunk division (the generic i / nvec form cost 1.4 us of
// issue time per 47-row tile).
__device__ __forceinline__ void kv_copy_tile(uint32_t kd, uint32_t vd, const __half* ks, const __half* vs, int nr,
                                             int dhp, int swz) {
    const int nvec = dhp >> 3, tid = threadIdx.x;
    if (nvec <= kConsumers && kConsumers % nvec == 0) {
        const int rstep = kConsumers / nvec, c = tid % nvec;
#pragma unroll 2
        for (int r = tid / nvec; r < nr; r += rstep) {
            const uint32_t o = kv_chunk_off(r, c, dhp, swz);
            const size_t g = (size_t)r * dhp + c * 8;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(kd + o), "l"(ks + g));
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(vd + o), "l"(vs + g));
        }
    } else {
        for (int i = tid; i < nr * nvec; i += kConsumers) {
            const int r = i / nvec, c = i - r * nvec;
            const uint32_t o = kv_chunk_off(r, c, dhp, swz);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(kd + o), "l"(ks + i * 8));
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(vd + o), "l"(vs + i * 8));
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

__device__ __noinline__ void attn_scores(uint32_t kt, int dhp, int swz, int nrb, int nr, uint32_t qh_s, float* sc, float scale2) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int npair = dhp >> 4;
    if (warp < nrb) {
        float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};
        const int mi = lane >> 3;
        const int arow_i = warp * 16 + (lane & 7) + ((mi & 1) << 3);
        const uint32_t arow = kt + arow_i * dhp * 2;
        const int axor = arow_i & swz, ahi = mi >> 1;
#pragma unroll 2
        for (int ks = 0; ks < npair; ++ks) {
            uint32_t a[4];
            ldsm4(a, arow + (((2 * ks + ahi) ^ axor) << 4));
            uint32_t b0 = 0u, b1 = 0u;
            if (lane < 4) {
                asm("ld.shared.u32 %0, [%1];" : "=r"(b0) : "r"(qh_s + (ks * 16 + 2 * lane) * 2));
                asm("ld.shared.u32 %0, [%1];" : "=r"(b1) : "r"(qh_s + (ks * 16 + 8 + 2 * lane) * 2));
            }
            if (ks & 1) mma_16816(c1, a, b0, b1); else mma_16816(c0, a, b0, b1);
        }
        if ((lane & 3) == 0) {
            const int rlo = warp * 16 + (lane >> 2), rhi = rlo + 8;
            sc[rlo] = (rlo < nr) ? h2f_round(h2f_round(c0[0] + c1[0]) * scale2) : -INFINITY;
            sc[rhi] = (rhi < nr) ? h2f_round(h2f_round(c0[2] + c1[2]) * scale2) : -INFINITY;
        }
    }
}

// attention output of one (sample, head): dims d, d+1 as one LL word of the `a` buffer
__device__ __forceinline__ void attn_out_pair(const EngineDev* E, int b, int h, int d, float v0, float v1, uint32_t flag) {
    const __half2 o = __floats2half2_rn(v0, v1);
    ll_st(E->ll_a + (((size_t)b * E->S + h * E->dh + d) >> 1), *reinterpret_cast<const uint32_t*>(&o), flag);
}

// One (sample, head, part) work item; q_len == 1 (reference factored_attention.py:82-133 and the
// per-pattern sample branches :135-228).
//   * q and the current token's k, v come from the QKV Conv1D as LL words (polled: this is the QKV -> attention
//     hand-over); the part's cached K and V rows are staged with cp.async into swizzled tiles, issued BEFORE the
//     poll so their HBM latency overlaps it; a part that fits one tile (RC-1 cached rows + the current token) is
//     ONE tile, longer parts (dense / prime / enc-dec layers) run double-buffered through both tile regions
//   * scores on the tensor cores: A = 16 key rows x 16 dims (ldmatrix), B = q in column 0, fp32
//     accumulate; s = fp16(fp16(q.k) * dh^-1/2) exactly as the reference rounds it
//   * softmax is flash-style in fp32 (running max / sum), every warp redundantly; P rounded to fp16 as
//     the reference's w.half(), P.V on the tensor cores (A = P in row 0, B = V via ldmatrix.trans), each
//     warp owning 16-dim output slices
//   * parts 0 .. ns-2 of one (sample, head) publish their (max, sum, output) as LL words; the last part, which also
//     holds the current token, polls them and merges (flash-decoding merge); the output goes to the `a` LL buffer,
//     which IS the attention -> proj hand-over
__device__ __noinline__ void attn_item(const LayerDev& LD_ref, int b, int h, int s, int ns,
                                       const AttnGeom G, int pslot, uint32_t flag, int pre) {
    const EngineDev* E = sm_E();
    uint8_t* uni = sm_uni();
    const LayerDev LD = LD_ref;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int dh = E->dh, dhp = E->dh_pad, S = E->S;
    const int nvec = dhp >> 3, npair = dhp >> 4;
    const int swz = (nvec & 7) ? 0 : 7;
    const int RC = E->RC;
    const int tileB = RC * dhp * 2;
    // two tile regions; a prefetched first tile (attn_prefetch) sits in the second one, which no other phase touches
    const uint32_t regU = smem_u32(uni), regX = smem_u32(jk_smem + kHeaderBytes + E->uni_bytes);
    const uint32_t regA = pre ? regX : regU, regB = pre ? regU : regX;
    __half* qh = reinterpret_cast<__half*>(uni + 2 * tileB);          // [dhp] q, then [dhp] k_new, [dhp] v_new
    __half* kn = qh + dhp;
    __half* vn = kn + dhp;
    float* sc = reinterpret_cast<float*>(uni + 2 * tileB + 3 * dhp * 2);  // [64] scores of the tile
    const int qkv_words = ((LD.attn_func == 6) ? S : 3 * S) >> 1;
    const unsigned long long* qrow = E->ll_qkv + (size_t)b * qkv_words + ((h * dh) >> 1);
    const size_t cbase = ((size_t)(b * E->H + h)) * LD.rows;
    const bool last_part = (s == ns - 1);
    const int R = G.R;
    const int ncache = R - ((R > 0 && G.cur) ? 1 : 0);               // rows that come from the cache
    const int i0 = div_small(ncache * s, ns), i1 = div_small(ncache * (s + 1), ns);
    const __half* kbase = LD.kc + (cbase + G.base) * dhp;
    const __half* vbase = LD.vc + (cbase + G.base) * dhp;
    const int trows = RC - 1;
    const int ntiles = max(1, (i1 - i0 + trows - 1) / trows);

    auto issue_tile = [&](int ti) {
        const int r0 = i0 + ti * trows, nr = max(0, min(trows, i1 - r0));
        const uint32_t kd = (ti & 1) ? regB : regA, vd = kd + tileB;
        kv_copy_tile(kd, vd, kbase + (size_t)r0 * dhp, vbase + (size_t)r0 * dhp, nr, dhp, swz);
    };
    STAMP(E, pslot, 0);
    if (R > 0 && !pre) issue_tile(0);       // cached rows do not depend on the current token: load them first
    // ---- q, k_new, v_new of this (sample, head): LL words of the QKV Conv1D, polled --------------------------
    {
        const int hw = dhp >> 1, dw = dh >> 1;
        const int nsel = (LD.attn_func == 6) ? 1 : 3;
        // up to three words per thread (dh <= 512), ALL issued before the first is examined: one L2 round trip, where a
        // loop of blocking polls paid one per iteration (two for head_dim 256)
        const int total = nsel * hw;
        unsigned long long wv[3];
        const unsigned long long* wp[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int i = tid + j * kConsumers;
            const int sel = (i >= hw) + (i >= 2 * hw), wd = i - sel * hw;
            wp[j] = (i < total && wd < dw) ? qrow + (size_t)sel * (S >> 1) + wd : nullptr;
            if (wp[j]) wv[j] = ll_ld1(wp[j]);
        }
        unsigned spins = 0;
        for (;;) {
            bool again = false;
#pragma unroll
            for (int j = 0; j < 3; ++j)
                if (wp[j] && !ll_ok(wv[j], flag)) { wv[j] = ll_ld1(wp[j]); again = true; }
            if (!again) break;
            spin_guard(spins);
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int i = tid + j * kConsumers;
            if (i < total) reinterpret_cast<uint32_t*>(qh)[i] = wp[j] ? (uint32_t)wv[j] : 0u;
        }
    }
    consumer_sync();
    if (G.wrow >= 0 && last_part) {          // cache the current token's k, v
        for (int i = tid; i < dh; i += kConsumers) {
            LD.kc[(cbase + G.wrow) * dhp + i] = kn[i];
            LD.vc[(cbase + G.wrow) * dhp + i] = vn[i];
        }
    }
    if (R == 0) {   // prev-block attention inside the first block: keys/values are zeros -> output 0
        if (2 * tid < dh) attn_out_pair(E, b, h, 2 * tid, 0.f, 0.f, flag);
        return;
    }

    float m_run = -INFINITY, l_run = 0.f;
    float* osm = sc + 64;                                  // [dhp] running output of multi-tile parts (owner-private)
    const uint32_t qh_s = smem_u32(qh);
#pragma unroll 1
    for (int ti = 0; ti < ntiles; ++ti) {
        if (ti + 1 < ntiles) {
            issue_tile(ti + 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        const int r0 = i0 + ti * trows;
        int nr = max(0, min(trows, i1 - r0));
        const uint32_t kt = (ti & 1) ? regB : regA, vt = kt + tileB;
        if (ti == ntiles - 1 && last_part && G.cur) {       // append the current token's k, v (from the QKV GEMM)
            for (int c8 = tid; c8 < nvec; c8 += kConsumers) {
                const uint32_t o = kv_chunk_off(nr, c8, dhp, swz);
                const uint4 kq = *reinterpret_cast<const uint4*>(kn + c8 * 8), vq = *reinterpret_cast<const uint4*>(vn + c8 * 8);
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(kt + o), "r"(kq.x), "r"(kq.y), "r"(kq.z), "r"(kq.w));
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(vt + o), "r"(vq.x), "r"(vq.y), "r"(vq.z), "r"(vq.w));
            }
            nr += 1;
        }
        const int nrb = (nr + 15) >> 4;                     // 16-row blocks of this tile
        // V rows past nr inside the last row block meet P = 0 in the MMA: they must be finite
        for (int i = tid; i < (nrb * 16 - nr) * nvec; i += kConsumers) {
            const int r = nr + i / nvec, c = i % nvec;
            asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(vt + kv_chunk_off(r, c, dhp, swz)), "r"(0u));
        }
        consumer_sync();
        STAMP(E, pslot, 1);
        // ---- scores: warp w < nrb owns key rows [16w, 16w+16) ----------------------------------------
        attn_scores(kt, dhp, swz, nrb, nr, qh_s, sc, E->scale2);
        consumer_sync();
        STAMP(E, pslot, 2);
        // ---- softmax of the tile (every warp, redundantly): lane r holds rows r and r + 32 -------------
        const float s0 = (lane < nrb * 16) ? sc[lane] : -INFINITY;
        const float s1 = (lane + 32 < nrb * 16) ? sc[lane + 32] : -INFINITY;
        const float m_new = fmaxf(m_run, warp_max(fmaxf(s0, s1)));
        const float corr = expf(m_run - m_new);              // exp(-inf) = 0 on the first tile
        const float p0 = expf(s0 - m_new), p1 = expf(s1 - m_new);
        l_run = l_run * corr + warp_sum(p0 + p1);
        m_run = m_new;
        // ---- P.V: this warp's 16-dim output slices, all row blocks.  A = P (fp16) in row 0 --------------
        {
            uint32_t pa0[4], pa2[4];
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const float src = (ks < 2) ? p0 : p1;
                const int l0 = (ks & 1) * 16 + 2 * (lane & 3);
                const float pa = __shfl_sync(0xffffffffu, src, l0), pb = __shfl_sync(0xffffffffu, src, l0 + 1);
                const float pc = __shfl_sync(0xffffffffu, src, l0 + 8), pd = __shfl_sync(0xffffffffu, src, l0 + 9);
                const __half2 h0 = __floats2half2_rn(pa, pb), h2 = __floats2half2_rn(pc, pd);
                pa0[ks] = (lane < 4) ? *reinterpret_cast<const uint32_t*>(&h0) : 0u;
                pa2[ks] = (lane < 4) ? *reinterpret_cast<const uint32_t*>(&h2) : 0u;
            }
            const int mi = lane >> 3;
            const int vrow_l = (lane & 7) + ((mi & 1) << 3), vhi = mi >> 1;
            const bool last_tile = (ti == ntiles - 1);
#pragma unroll 1
            for (int np = warp; np < npair; np += 8) {
                float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    if (ks < nrb) {
                        const int vrow_i = ks * 16 + vrow_l;
                        uint32_t bf[4];
                        ldsm4_trans(bf, vt + vrow_i * dhp * 2 + (((2 * np + vhi) ^ (vrow_i & swz)) << 4));
                        const uint32_t a[4] = {pa0[ks], 0u, pa2[ks], 0u};
                        mma_16816(o0, a, bf[0], bf[1]);
                        mma_16816(o1, a, bf[2], bf[3]);
                    }
                }
                if (lane < 4) {      // row 0: dims np*16 + {0, 8} + 2*lane, +1
                    const int d = np * 16 + 2 * lane;
                    float2 r0 = make_float2(o0[0], o0[1]), r1 = make_float2(o1[0], o1[1]);
                    if (ti > 0) {
                        const float2 q0 = *reinterpret_cast<const float2*>(osm + d), q1 = *reinterpret_cast<const float2*>(osm + d + 8);
                        r0.x += q0.x * corr; r0.y += q0.y * corr; r1.x += q1.x * corr; r1.y += q1.y * corr;
                    }
                    if (!last_tile) {
                        *reinterpret_cast<float2*>(osm + d) = r0;
                        *reinterpret_cast<float2*>(osm + d + 8) = r1;
                    } else if (ns == 1) {
                        const float inv = 1.f / l_run;
                        if (d < dh) attn_out_pair(E, b, h, d, r0.x * inv, r0.y * inv, flag);
                        if (d + 8 < dh) attn_out_pair(E, b, h, d + 8, r1.x * inv, r1.y * inv, flag);
                    } else if (last_part) {    // the merging part keeps its own partial in shared memory (osm is free now)
                        *reinterpret_cast<float2*>(osm + d) = r0;
                        *reinterpret_cast<float2*>(osm + d + 8) = r1;
                    } else {                   // the others publish theirs as LL words {fp32, flag}
                        unsigned long long* pl = E->part + ((size_t)((b * E->H + h) * kMaxSplit + s)) * (dhp + 2) + 2 + d;
                        const unsigned long long fw = (unsigned long long)flag << 32;
                        asm volatile(JK_ST_LL ".v2.u64 [%0], {%1,%2};" ::"l"(pl), "l"(fw | __float_as_uint(r0.x)),
                                     "l"(fw | __float_as_uint(r0.y)) : "memory");
                        asm volatile(JK_ST_LL ".v2.u64 [%0], {%1,%2};" ::"l"(pl + 8), "l"(fw | __float_as_uint(r1.x)),
                                     "l"(fw | __float_as_uint(r1.y)) : "memory");
                    }
                }
            }
        }
        if (ti + 1 < ntiles) consumer_sync();                 // tile buffers and sc are reused
    }
    STAMP(E, pslot, 3);
    if (ns == 1) return;
    // ---- split parts: parts 0 .. ns-2 publish (m, l, o) as LL words; the LAST part (the one that also holds the current
    // token) polls them and merges - a fixed merger: no ticket atomic (an acq_rel round trip), no second barrier, and the
    // partials arrive word by word like every other hand-over.  Summed in part order 0 .. ns-1: bit-reproducible.
    unsigned long long* pbase = E->part + ((size_t)((b * E->H + h) * kMaxSplit)) * (dhp + 2);
    if (!last_part) {
        if (tid == 0) {
            const unsigned long long fw = (unsigned long long)flag << 32;
            asm volatile(JK_ST_LL ".v2.u64 [%0], {%1,%2};" ::"l"(pbase + (size_t)s * (dhp + 2)), "l"(fw | __float_as_uint(m_run)),
                         "l"(fw | __float_as_uint(l_run)) : "memory");
        }
        STAMP(E, pslot, 6);
        return;
    }
    consumer_sync();                       // every warp's slice of this part's output is in osm
    const int d = 2 * tid;
    if (d < dh) {
        ulonglong2 ml[3], vv[3];
        unsigned spins = 0;
        bool again;
        do {
            again = false;
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                if (q < ns - 1) {
                    ml[q] = ll_ld2(pbase + (size_t)q * (dhp + 2));
                    vv[q] = ll_ld2(pbase + (size_t)q * (dhp + 2) + 2 + d);
                }
            }
#pragma unroll
            for (int q = 0; q < 3; ++q)
                if (q < ns - 1) again |= !(ll_ok(ml[q].x, flag) && ll_ok(ml[q].y, flag) && ll_ok(vv[q].x, flag) && ll_ok(vv[q].y, flag));
            if (again) spin_guard(spins);
        } while (again);
        float M = m_run;
#pragma unroll
        for (int q = 0; q < 3; ++q)
            if (q < ns - 1) M = fmaxf(M, __uint_as_float((uint32_t)ml[q].x));
        float Lsum = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            if (q < ns - 1) {
                const float w = expf(__uint_as_float((uint32_t)ml[q].x) - M);
                Lsum += __uint_as_float((uint32_t)ml[q].y) * w;
                o0 += __uint_as_float((uint32_t)vv[q].x) * w; o1 += __uint_as_float((uint32_t)vv[q].y) * w;
            }
        }
        {
            const float w = expf(m_run - M);
            const float2 own = *reinterpret_cast<const float2*>(osm + d);
            Lsum += l_run * w; o0 += own.x * w; o1 += own.y * w;
        }
        attn_out_pair(E, b, h, d, o0 / Lsum, o1 / Lsum, flag);
    }
    STAMP(E, pslot, 6);
}

// The cached K/V rows of this CTA's first attention item do not depend on the current token: issue their cp.async BEFORE
// the layer's QKV Conv1D, into the tile region that only the attention phase uses, so that the HBM latency hides behind
// that phase.  Returns 1 if the tile is on its way.
__device__ __noinline__ int attn_prefetch(const LayerDev& LD_ref, int B, int c, int t, int pm, int pd, int gmax) {
    const EngineDev* E = sm_E();
    const LayerDev LD = LD_ref;
    const AttnGeom G = attn_geom(E, LD, t, pm, pd);
    if (G.R == 0) return 0;
    const int ncache = G.R - (G.cur ? 1 : 0);
    const int ns = attn_nsplit(E, gmax, ncache);
    if (c >= B * E->H * ns) return 0;
    const int bh = div_small(c, ns), s = c - bh * ns, b = bh / E->H, h = bh - b * E->H;
    const int dhp = E->dh_pad, nvec = dhp >> 3, RC = E->RC;
    const int swz = (nvec & 7) ? 0 : 7;
    const int i0 = div_small(ncache * s, ns), i1 = div_small(ncache * (s + 1), ns);
    const int nr = max(0, min(RC - 1, i1 - i0));
    const size_t cbase = ((size_t)(b * E->H + h)) * LD.rows;
    const uint32_t kd = smem_u32(jk_smem + kHeaderBytes + E->uni_bytes), vd = kd + RC * dhp * 2;
    kv_copy_tile(kd, vd, LD.kc + (cbase + G.base + i0) * dhp, LD.vc + (cbase + G.base + i0) * dhp, nr, dhp, swz);
    return 1;
}

// ---------------------------------------------------------------------------------------
// producer warp: walks this CTA's weight stream (and the logits rows) in consumption order
// ---------------------------------------------------------------------------------------
template <int R>
__device__ __noinline__ void producer_loop(const EngineDev* E, Ring ring, int do_logits, int c) {
    if ((threadIdx.x & 31) != 0) return;
    const uint8_t* src = E->streams + (size_t)c * E->stream_stride;
    const int KS = E->KS, u = c >> E->ks_shift;
    for (int l = 0; l < E->depth; ++l) {
        const ushort2* cl = E->cols + ((size_t)u * E->depth + l) * 4;
        const int Ks[4] = {E->W >> E->ks_shift, E->S >> E->ks_shift, E->W >> E->ks_shift, E->M >> E->ks_shift};
        if (c == (l % E->G)) {
            // biases + LayerNorm parameters of this layer (one contiguous block, ~57 KB for 1b_lyrics) are
            // shared by every CTA and evicted from L2 between steps: pull them into L2 ahead of the consumers
            // (this producer runs about a layer ahead of them)
            const char* p0 = reinterpret_cast<const char*>(E->layer[l].b_qkv);
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p0), "r"((uint32_t)E->small_bytes) : "memory");
        }
#pragma unroll
        for (int gi = 0; gi < 4; ++gi) {
            const int ncg = cl[gi].y;
            if (ncg == 0) continue;
            const int nkk = Ks[gi] >> 4, kpc = kpc_of(ncg);
            for (int kk0 = 0; kk0 < nkk; kk0 += kpc) {
                const int nk = min(kpc, nkk - kk0);
                const uint32_t bytes = (uint32_t)nk * ncg * 256u;
                mbar_wait(ring.empty(), ring.phase ^ 1u);
                mbar_expect_tx(ring.full(), bytes);
                tma_bulk_g2s(ring.data(), src, bytes, ring.full());
                src += bytes;
                ring.advance();
            }
        }
    }
    if (do_logits == 2) {       // logits GEMM: one more Conv1D per pass in the stream
        for (int p = 0; p < E->lg_np; ++p) {
            const int ncg = E->lg_cols[p * E->U + u].y;
            if (ncg == 0) continue;
            const int nkk = ((2 * E->W) >> E->ks_shift) >> 4, kpc = kpc_of(ncg);
            for (int kk0 = 0; kk0 < nkk; kk0 += kpc) {
                const int nk = min(kpc, nkk - kk0);
                const uint32_t bytes = (uint32_t)nk * ncg * 256u;
                mbar_wait(ring.empty(), ring.phase ^ 1u);
                mbar_expect_tx(ring.full(), bytes);
                tma_bulk_g2s(ring.data(), src, bytes, ring.full());
                src += bytes;
                ring.advance();
            }
        }
    } else if (do_logits) {
        const int r0 = E->lrow0[c], r1 = E->lrow0[c + 1];
        const int W = E->W;
        for (int pr = r0; pr < r1; pr += kLogitRowsPerPass) {
            const int pe = min(r1, pr + kLogitRowsPerPass);
            for (int k0 = 0; k0 < W; k0 += logit_kt(R)) {
                const int kt = min(logit_kt(R), W - k0);
                for (int r = pr; r < pe; r += kLogitRowsPerChunk) {
                    const int nr = min(kLogitRowsPerChunk, pe - r);
                    mbar_wait(ring.empty(), ring.phase ^ 1u);
                    mbar_expect_tx(ring.full(), (uint32_t)(nr * kt * 4));
                    for (int i = 0; i < nr; ++i)
                        tma_bulk_g2s(ring.data() + i * kt * 4, E->x_out + (size_t)(r + i) * W + k0,
                                     (uint32_t)(kt * 4), ring.full());
                    ring.advance();
                }
            }
        }
    }
}

// fp32 logits: logits[b, r] = sum_k y[b, k] * x_out[r, k],  y = float(h) (+ cond)
// (reference autoregressive.py:226-229: fp32 nn.Linear on the fp32 transformer output)
// Warp w owns the sample rows [w * R / 8, (w + 1) * R / 8): every x_out row is streamed once whatever R.
template <int R>
__device__ __noinline__ void logits_phase(const StepArgs& A_ref, Ring& ring_ref, int c, int t, uint32_t flag) {
    constexpr int RPW = R / 8;                      // sample rows per warp: 2 or 4
    const EngineDev* E = sm_E();
    uint8_t* uni = sm_uni();
    const StepArgs A = A_ref;
    Ring ring = ring_ref;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int r0 = E->lrow0[c], r1 = E->lrow0[c + 1];
    const int W = E->W, B = A.n;
    float* ys = reinterpret_cast<float*>(uni);     // [R][kt]
    for (int pr = r0; pr < r1; pr += kLogitRowsPerPass) {
        const int pe = min(r1, pr + kLogitRowsPerPass);
        float acc[kLogitRowsPerPass][RPW];
#pragma unroll
        for (int i = 0; i < kLogitRowsPerPass; ++i) acc[i][0] = acc[i][1] = 0.f;
        if constexpr (RPW == 4) {
#pragma unroll
            for (int i = 0; i < kLogitRowsPerPass; ++i) acc[i][2] = acc[i][3] = 0.f;
        }
        for (int k0 = 0; k0 < W; k0 += logit_kt(R)) {
            const int kt = min(logit_kt(R), W - k0);
            consumer_sync();
            {   // y = float(h) (+ cond): the final residual stream as LL words, 4 halves per 16-byte polled load
                const int nv = kt >> 2;
                for (int idx0 = tid; idx0 < R * nv; idx0 += 4 * kConsumers) {
                    ulonglong2 hv[4];
                    unsigned spins = 0;
                    bool again;
                    do {
                        again = false;
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const int idx = idx0 + u * kConsumers;
                            const int b = idx / nv, v = idx - b * nv;
                            if (idx < R * nv && b < B) {
                                hv[u] = ll_ld2(E->ll_h + (((size_t)b * W + k0 + v * 4) >> 1));
                                again |= !(ll_ok(hv[u].x, flag) && ll_ok(hv[u].y, flag));
                            }
                        }
                        if (again) spin_guard(spins);
                    } while (again);
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int idx = idx0 + u * kConsumers;
                        if (idx >= R * nv) continue;
                        const int b = idx / nv, v = idx - b * nv;
                        float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (b < B) {
                            const uint32_t lo = (uint32_t)hv[u].x, hi = (uint32_t)hv[u].y;
                            const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&lo));
                            const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&hi));
                            y = make_float4(f0.x, f0.y, f1.x, f1.y);
                            if (E->add_cond_after && A.x_cond) {
                                const float* cp = A.x_cond + ((size_t)b * A.x_cond_len + (A.x_cond_len > 1 ? t : 0)) * W + k0 + v * 4;
                                const float4 c0 = *reinterpret_cast<const float4*>(cp);
                                y.x += c0.x; y.y += c0.y; y.z += c0.z; y.w += c0.w;
                            }
                        }
                        *reinterpret_cast<float4*>(ys + b * kt + v * 4) = y;
                    }
                }
            }
            consumer_sync();
            const float* y0 = ys + (warp * RPW) * kt;
            const float* y1 = y0 + kt;
#pragma unroll
            for (int rc = 0; rc < kLogitRowsPerPass / kLogitRowsPerChunk; ++rc) {
                const int r = pr + rc * kLogitRowsPerChunk;
                if (r < pe) {
                    const int nr = min(kLogitRowsPerChunk, pe - r);
                    mbar_wait(ring.full(), ring.phase);
                    const float* wsl = reinterpret_cast<const float*>(ring.data());
#pragma unroll 1
                    for (int k = lane * 4; k < kt; k += 128) {      // rolled: this phase runs once per step, its code must stay small
                        float4 a0 = *reinterpret_cast<const float4*>(y0 + k);
                        float4 a1 = *reinterpret_cast<const float4*>(y1 + k);
                        float4 a2, a3;
                        if constexpr (RPW == 4) {
                            a2 = *reinterpret_cast<const float4*>(y1 + kt + k);
                            a3 = *reinterpret_cast<const float4*>(y1 + 2 * kt + k);
                        }
#pragma unroll
                        for (int i = 0; i < kLogitRowsPerChunk; ++i) {
                            if (i < nr) {
                                float4 w4 = *reinterpret_cast<const float4*>(wsl + i * kt + k);
                                acc[rc * kLogitRowsPerChunk + i][0] += a0.x * w4.x + a0.y * w4.y + a0.z * w4.z + a0.w * w4.w;
                                acc[rc * kLogitRowsPerChunk + i][1] += a1.x * w4.x + a1.y * w4.y + a1.z * w4.z + a1.w * w4.w;
                                if constexpr (RPW == 4) {
                                    acc[rc * kLogitRowsPerChunk + i][2] += a2.x * w4.x + a2.y * w4.y + a2.z * w4.z + a2.w * w4.w;
                                    acc[rc * kLogitRowsPerChunk + i][3] += a3.x * w4.x + a3.y * w4.y + a3.z * w4.z + a3.w * w4.w;
                                }
                            }
                        }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(ring.empty());
                    ring.advance();
                }
            }
        }
#pragma unroll
        for (int i = 0; i < kLogitRowsPerPass; ++i) {
            float v0 = warp_sum(acc[i][0]), v1 = warp_sum(acc[i][1]), v2 = 0.f, v3 = 0.f;
            if constexpr (RPW == 4) { v2 = warp_sum(acc[i][2]); v3 = warp_sum(acc[i][3]); }
            const int r = pr + i;
            if (lane == 0 && r < pe) {
                const int b0 = warp * RPW;
                if (b0 < B) A.logits[(size_t)b0 * A.logits_bstride + (size_t)t * A.logits_tstride + r] = v0;
                if (b0 + 1 < B) A.logits[(size_t)(b0 + 1) * A.logits_bstride + (size_t)t * A.logits_tstride + r] = v1;
                if constexpr (RPW == 4) {
                    if (b0 + 2 < B) A.logits[(size_t)(b0 + 2) * A.logits_bstride + (size_t)t * A.logits_tstride + r] = v2;
                    if (b0 + 3 < B) A.logits[(size_t)(b0 + 3) * A.logits_bstride + (size_t)t * A.logits_tstride + r] = v3;
                }
            }
        }
    }
}

// Housekeeping of the LayerNorm statistics blocks, on warp 9 of CTA 0 (a warp of the producer warpgroup that has nothing
// else to do).  Block i (0 .. 2 * depth) is used once per launch and must be zero again at the next launch.  It may be
// cleared once a LATER block is complete: every CTA contributes to block i + 1 only after it has consumed block i
// (program order + data dependence).  On the consumer warps of CTA 0 this would put a polled L2 round trip on the
// critical path of CTA 0 (and so of its unit) twice per layer.  The same warp publishes the position and the step count
// at the end: the final block is complete only when every CTA is through the stack, and every CTA has read both words
// long before that.
// Lane l clears word l & 1 of rows l / 2 (+ 16): the R rows a launch of R rows adds to.
template <int R>
__device__ __noinline__ void cleaner_loop() {
    const EngineDev* E = sm_E();
    const int lane = threadIdx.x & 31, G = E->G, nblk = 2 * E->depth;
    const int t = *reinterpret_cast<volatile const int*>(E->t);
    const unsigned step = *reinterpret_cast<volatile const unsigned*>(E->step);
    for (int i = 1; i <= nblk; ++i) {
        if (lane == 0) wait_stat_word(E->lnacc + (size_t)i * 512, G);
        __syncwarp();
#pragma unroll
        for (int r = 0; r < R; r += 16) (E->lnacc + (size_t)(i - 1) * 512)[16 * (r + (lane >> 1)) + (lane & 1)] = 0;
    }
#pragma unroll
    for (int r = 0; r < R; r += 16) (E->lnacc + (size_t)nblk * 512)[16 * (r + (lane >> 1)) + (lane & 1)] = 0;
    if (lane == 0) {
        *E->t = t + 1;
        *E->step = step + 1;
    }
}

// ---------------------------------------------------------------------------------------
// Values of a launch that every phase call would otherwise have to keep in a register: ptxas allocates the __noinline__
// phases inter-procedurally, so each value live across the calls is a register less inside them (on sm_90a, keeping
// these in registers made gemm_phase spill).  The descriptor fields are re-read from its shared-memory copy; the position,
// its block coordinates and the step count live in the header's LaunchVals, written by the kernel prologue.
__device__ __forceinline__ int launch_pos() { return sm_launch()->t; }
__device__ __forceinline__ int launch_pm() { return sm_launch()->pm; }
__device__ __forceinline__ int launch_pd() { return sm_launch()->pd; }
__device__ __forceinline__ int launch_gmax() { return sm_launch()->gmax; }
__device__ __forceinline__ uint32_t launch_step() { return sm_launch()->step; }
// LL flags of this launch: launch_fbase() + 1 .. launch_fbase() + depth + 1
__device__ __forceinline__ uint32_t launch_fbase() { return launch_step() * (uint32_t)(sm_E()->depth + 2); }
__device__ __forceinline__ int cta_unit() { return (int)blockIdx.x >> sm_E()->ks_shift; }
__device__ __forceinline__ int cta_rank() { return (int)blockIdx.x & (sm_E()->KS - 1); }
__device__ __forceinline__ bool wants_logits(const StepArgs& A) { return A.logits != nullptr && sm_E()->bins > 0; }
// y = h + x_cond is not an fp16 value: those configurations (upsamplers) keep the fp32 FMA path (unless the caller supplies
// x_cond . x_out^T, the logit bias of jkb200.h: the product is linear in the activation)
__device__ __forceinline__ bool logits_on_mma(const StepArgs& A) {
    const EngineDev* E = sm_E();
    return E->lg_on && (!(E->add_cond_after && A.x_cond) || A.logit_bias);
}

template <int R>
__global__ void __launch_bounds__(kThreads, 1) jk_decode_step_kernel(const EngineDev* __restrict__ Eg, StepArgs A) {
    const int tid = threadIdx.x, warp = tid >> 5;
    const int c = blockIdx.x;
    for (int i = tid; i < (int)(offsetof(EngineDev, layer) / 4); i += kThreads)
        sm_desc_words()[i] = reinterpret_cast<const uint32_t*>(Eg)[i];
    if (tid < (int)(sizeof(LayerDev) / 4))
        reinterpret_cast<uint32_t*>(sm_layer_slot(0))[tid] = reinterpret_cast<const uint32_t*>(&Eg->layer[0])[tid];
    __syncthreads();
    const EngineDev* E = sm_E();
    if (tid >= 32 && tid < 36)
        reinterpret_cast<uint32_t*>(sm_cols(0))[tid - 32] =
            reinterpret_cast<const uint32_t*>(E->cols + ((size_t)cta_unit() * E->depth + 0) * 4)[tid - 32];
    Ring ring;
    ring.slot = 0; ring.phase = 0;
    if (tid == 0) {
        for (int i = 0; i < E->nslot; ++i) { mbar_init(sm_full() + i, 1); mbar_init(sm_empty() + i, 8); }
        mbar_fence_init();
    }
    __syncthreads();
    // Register reallocation between warpgroups (setmaxnreg, sm_90a+): the block launches with 168 registers per
    // thread (65536 / 384); the producer warpgroup keeps 40 and hands the rest to the two consumer warpgroups.
    if (warp >= 8) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8) producer_loop<R>(Eg, ring, wants_logits(A) ? (logits_on_mma(A) ? 2 : 1) : 0, c);
        else if (warp == 9 && c == 0) cleaner_loop<R>();
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int B = A.n;
    // per-launch values live in shared memory (not in registers across the phase calls)
    if (tid == 0) {
        LaunchVals* lv = sm_launch();
        const int t = *reinterpret_cast<volatile const int*>(E->t);
        lv->pm = E->blocks > 0 ? t % E->bc : 0;
        lv->pd = E->blocks > 0 ? t / E->bc : 0;
        lv->gmax = max(1, E->G / (B * E->H));
        lv->t = t;
        // written only at the very end of a launch by CTA 0, after every CTA of that launch has passed an all-to-all
        // point - so every CTA of this launch reads the same value
        lv->step = *reinterpret_cast<volatile const unsigned*>(E->step);
    }
    // thread layouts of the activation staging for the three K of a layer (integer divisions: once per launch, not per phase)
    stage_map_init(0, E->W >> E->ks_shift);
    stage_map_init(1, E->S >> E->ks_shift);
    stage_map_init(2, E->M >> E->ks_shift);
    consumer_sync();
    unsigned nph = 0;                                             // phase index (profiling slots)
#define PHASE_DONE()                                                                           \
    do {                                                                                       \
        ++nph;                                                                                 \
        if (c == 0 && tid == 0 && E->prof_on && nph < (unsigned)kProfSlots) {                  \
            unsigned long long now;                                                            \
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));                            \
            E->prof[nph] = now;                                                                \
        }                                                                                      \
    } while (0)
#define PROF3(idx_, which_)                                                                    \
    do {                                                                                       \
        if (tid == 0 && E->prof_on) {                                                          \
            unsigned long long now_;                                                           \
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now_));                           \
            E->prof3[((idx_) * 256 + c) * 2 + (which_)] = now_;                                \
        }                                                                                      \
    } while (0)
    if (c == 0 && tid == 0 && E->prof_on) {
        unsigned long long now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        E->prof[0] = now;
    }

    // ---- P0: embedding (autoregressive.py:177-197) or an externally embedded activation ------
    // This CTA embeds exactly the columns of the residual stream it will own for the whole stack.
    {
        const ushort2 wc = sm_cols(0)[1];                   // column groups of width-W outputs
        const int ppc = (wc.y * 4) >> E->ks_shift;
        long long* sfx = sm_sfx<R>();
        const int lane = tid & 31;
        for (int b = warp; b < B && lane < ppc; b += 8) {     // lane = column pair, warp = sample row (and row + 8, ...)
            const int pl = lane;
            const int col = wc.x * 8 + 2 * (cta_rank() * ppc + pl);
            float2 x;
            if (A.x_in) {
                x = *reinterpret_cast<const float2*>(A.x_in + (size_t)b * E->W + col);
            } else {
                if (launch_pos() == 0) x = A.y_cond ? *reinterpret_cast<const float2*>(A.y_cond + (size_t)b * E->W + col)
                                         : *reinterpret_cast<const float2*>(E->start_token + col);
                else x = *reinterpret_cast<const float2*>(E->x_emb + (size_t)A.tokens[(size_t)b * A.tok_stride + launch_pos() - 1] * E->W + col);
                const float2 pe = *reinterpret_cast<const float2*>(E->pos_emb + (size_t)launch_pos() * E->W + col);
                x.x += pe.x; x.y += pe.y;
                if (A.x_cond) {
                    const float2 xc = *reinterpret_cast<const float2*>(A.x_cond + ((size_t)b * A.x_cond_len + (A.x_cond_len > 1 ? launch_pos() : 0)) * E->W + col);
                    x.x += xc.x; x.y += xc.y;
                }
            }
            const __half2 hh = __floats2half2_rn(x.x, x.y);
            const float2 hv = __half22float2(hh);
            res_st<R>(b * 32 + pl, hv);
            sfx[b * 32 + pl] = fx_sum(hv.x) + fx_sum(hv.y);
            sfx[1024 + b * 32 + pl] = fx_sq(hv.x) + fx_sq(hv.y);
            ll_st(E->ll_h + (((size_t)b * E->W + col) >> 1), *reinterpret_cast<const uint32_t*>(&hh), launch_fbase() + 1);
        }
        publish_stats<R>(E->lnacc, B, ppc);     // statistics block 0: the input of layer 0's LN0
    }
    PHASE_DONE();

#pragma unroll 1
    for (int l = 0; l < E->depth; ++l) {
        const LayerDev& LD = *sm_layer(l);
        const uint32_t fl = launch_fbase() + (uint32_t)l + 1;              // flag of this layer's buffers
        const int pre = attn_prefetch(LD, B, c, launch_pos(), launch_pm(), launch_pd(), launch_gmax());
        // a fresh argument record per phase: nothing of it stays live across the calls in between
        if (l == 1) PROF3(0, 0);
        ring = gemm_phase<R>(ring, B, EPI_QKV, l, (int)nph, fl);
        if (l == 1) PROF3(0, 1);
        // next layer's record + column assignment -> the other shared-memory slot.  The descriptor is in
        // HBM (the weight stream evicts it from L2 every step): issue the loads here so their latency hides
        // behind the attention phase instead of sitting on the dependency chain.
        if (l + 1 < E->depth) {
            // cp.async: no register sits between the HBM load and the shared-memory store, so no warp stalls on it here;
            // it is waited for in front of this layer's last Conv1D (whose barriers publish it to the other threads)
            if (tid < (int)(sizeof(LayerDev) / 4))
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(sm_layer_slot(l + 1) + 4 * tid)),
                             "l"(reinterpret_cast<const uint32_t*>(&Eg->layer[l + 1]) + tid) : "memory");
            if (tid >= 32 && tid < 36)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(sm_cols(l + 1) + (tid - 32))),
                             "l"(reinterpret_cast<const uint32_t*>(E->cols + ((size_t)cta_unit() * E->depth + l + 1) * 4) + (tid - 32)) : "memory");
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        PHASE_DONE();
        if (l == 1) PROF3(1, 0);
        {
            const AttnGeom geo = attn_geom(E, LD, launch_pos(), launch_pm(), launch_pd());
            const int ns = attn_nsplit(E, launch_gmax(), geo.R - ((geo.R > 0 && geo.cur) ? 1 : 0));
            for (int it = c; it < B * E->H * ns; it += E->G) {
                const int bh = div_small(it, ns), s = it - bh * ns, ib = bh / E->H;
                attn_item(LD, ib, bh - ib * E->H, s, ns, geo, (int)nph, fl, pre && it == c);
                consumer_sync();           // tile / q regions are reused by the next item or the next phase
            }
        }
        if (l == 1) PROF3(1, 1);
        PHASE_DONE();
        if (l == 1) PROF3(2, 0);
        ring = gemm_phase<R>(ring, B, EPI_PROJ, l, (int)nph, fl);
        if (l == 1) PROF3(2, 1);
        PHASE_DONE();
        if (l == 1) PROF3(3, 0);
        ring = gemm_phase<R>(ring, B, EPI_FC, l, (int)nph, fl);
        if (l == 1) PROF3(3, 1);
        PHASE_DONE();
        if (l == 1) PROF3(4, 0);
        asm volatile("cp.async.wait_group 0;" ::: "memory");      // the next layer's record (issued a phase and a half ago)
        ring = gemm_phase<R>(ring, B, EPI_PROJ2, l, (int)nph, fl);
        if (l == 1) PROF3(4, 1);
        PHASE_DONE();
    }
    if (A.h_out) {      // Transformer.forward boundary: this CTA's slice of the residual stream
        const ushort2 wc = sm_cols(E->depth - 1)[1];
        const int ppc = (wc.y * 4) >> E->ks_shift;
        const int lane = tid & 31;
        for (int b = warp; b < B && lane < ppc; b += 8) {
            const int col = wc.x * 8 + 2 * (cta_rank() * ppc + lane);
            *reinterpret_cast<float2*>(A.h_out + (size_t)b * E->W + col) = res_ld<R>(b * 32 + lane);
        }
    }
    if (wants_logits(A) && logits_on_mma(A)) {
        // logits GEMM: [y | y] (the final residual stream, fp16-exact) x [hi(x_out) ; lo(x_out)] on the tensor cores, through
        // the same phase code as every Conv1D; the K-split partial sums (hi and lo halves on different ranks) meet in fp32.
        // Pass p exchanges its partial sums through xp[p], so no pass overwrites words the unit still polls for the pass
        // before it.  A CTA writes xp[p] (p >= 1) only after its epilogue of pass p - 1 has read the partials of every rank
        // of its unit: every CTA of the unit is then past the last layer, whose words in xp[p] have all been read.  Each
        // pass stages [y | y] again: the cross-warp reduction of the previous pass overwrote the tile.
        // The passes are unrolled (at most 4, compute_layout): a rolled loop around the call made ptxas spill in gemm_phase.
        stage_map_init(2, (2 * E->W) >> E->ks_shift);
        auto pass_record = [&](int p) {
            consumer_sync();
            if (tid == 0) {
                LogitsRec* lr = sm_lrec();
                lr->lg_out = A.logits + (size_t)launch_pos() * A.logits_tstride; lr->lg_bs = A.logits_bstride;
                lr->lb = (E->add_cond_after && A.x_cond) ? A.logit_bias + (size_t)launch_pos() * A.lb_tstride : nullptr; lr->lb_bs = A.lb_bstride;
                lr->cols = E->lg_cols[p * E->U + cta_unit()];
                lr->xp = E->xp[p];
            }
            consumer_sync();
        };
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            if (p < E->lg_np) {
                pass_record(p);
                ring = gemm_phase<R>(ring, B, EPI_LOGITS, E->depth - 1, (int)nph + p, launch_fbase() + (uint32_t)E->depth + 1);
            }
        }
    } else if (wants_logits(A)) {
        logits_phase<R>(A, ring, c, launch_pos(), launch_fbase() + (uint32_t)E->depth + 1);
    }
    if (c == 0) {
        consumer_sync();
        if (tid == 0) {
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (E->prof_on && nph + 1 < (unsigned)kProfSlots) E->prof[nph + 1] = now;
        }
    }
#undef PHASE_DONE
#undef PROF3
}

// ---------------------------------------------------------------------------------------
// packing kernels (one-time, at weight load)
// ---------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ __half to_half(T v);
template <>
__device__ __forceinline__ __half to_half<float>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __half to_half<__half>(__half v) { return v; }

// src: Conv1D.w [K][N] row-major.  dst: per-CTA streams; this kernel fills GEMM `gi` of layer `l`.
// grid.x = CTA index c = unit * KS + rank: the unit's column groups, the rank's K slice; threads loop over this
// CTA's (kk, j, lane) fragment slots.
template <typename T>
__global__ void pack_gemm_kernel(const T* __restrict__ src, int K, int N, uint8_t* streams,
                                 unsigned long long stream_stride, const ushort2* cols, const uint32_t* goff,
                                 int depth, int l, int gi, int KS) {
    const int c = blockIdx.x;
    const ushort2 cg = cols[((size_t)(c / KS) * depth + l) * 4 + gi];
    const int g0 = cg.x, ncg = cg.y;
    if (ncg == 0) return;
    uint8_t* dst = streams + (size_t)c * stream_stride + (size_t)goff[((size_t)c * depth + l) * 4 + gi] * 16;
    const int nkk = (K / KS) >> 4, kk_first = (c % KS) * nkk;
    const int total = nkk * ncg * 32;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const int lane = i & 31, u = i >> 5;
        const int j = u % ncg, kk = kk_first + u / ncg;
        const int n = (g0 + j) * 8 + (lane >> 2);
        const int k = kk * 16 + (lane & 3) * 2;
        __half v[4];
        v[0] = to_half<T>(src[(size_t)k * N + n]);
        v[1] = to_half<T>(src[(size_t)(k + 1) * N + n]);
        v[2] = to_half<T>(src[(size_t)(k + 8) * N + n]);
        v[3] = to_half<T>(src[(size_t)(k + 9) * N + n]);
        *reinterpret_cast<uint2*>(dst + (size_t)u * 256 + lane * 8) = *reinterpret_cast<uint2*>(v);
    }
}

// logits GEMM: x_out [bins][W] fp32 -> the same per-CTA fragment streams with K' = 2 W: rows k' < W hold hi = fp16(w),
// rows k' >= W hold lo = fp16(w - hi) (hi + lo carries 22 significant bits; y is an fp16 value, so y.hi + y.lo is the
// fp32 product up to 2^-22).  Appended to every CTA's stream after the last layer (lg_goff), one block per pass:
// grid (G, passes).
__global__ void pack_logits_kernel(const float* __restrict__ x_out, int W, int bins, uint8_t* streams,
                                   unsigned long long stream_stride, const ushort2* lg_cols, const uint32_t* lg_goff, int KS) {
    const int c = blockIdx.x, p = blockIdx.y, G = gridDim.x;
    const ushort2 cg = lg_cols[p * (G / KS) + c / KS];
    const int g0 = cg.x, ncg = cg.y;
    if (ncg == 0) return;
    uint8_t* dst = streams + (size_t)c * stream_stride + (size_t)lg_goff[p * G + c] * 16;
    const int nkk = ((2 * W) / KS) >> 4, kk_first = (c % KS) * nkk;
    const int total = nkk * ncg * 32;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const int lane = i & 31, u = i >> 5;
        const int j = u % ncg, kk = kk_first + u / ncg;
        const int n = (g0 + j) * 8 + (lane >> 2);
        const int k = kk * 16 + (lane & 3) * 2;
        const int ko[4] = {k, k + 1, k + 8, k + 9};
        __half v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const bool lo = ko[e] >= W;
            const float w = n < bins ? x_out[(size_t)n * W + (lo ? ko[e] - W : ko[e])] : 0.f;
            const __half hi = __float2half_rn(w);
            v[e] = lo ? __float2half_rn(w - __half2float(hi)) : hi;
        }
        *reinterpret_cast<uint2*>(dst + (size_t)u * 256 + lane * 8) = *reinterpret_cast<uint2*>(v);
    }
}

template <typename T>
__global__ void round_bias_kernel(const T* __restrict__ src, float* dst, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __half2float(to_half<T>(src[i]));
}
template <typename T>
__global__ void to_half_kernel(const T* __restrict__ src, __half* dst, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = to_half<T>(src[i]);
}

// encoder K/V for attn_func 6: kv = fp16(fp16(enc) . Wkv + b), once per window.  The product itself runs on
// the wgmma prefill GEMM (prefill_gemm.cu); these kernels only convert / lay out its operands and result.
template <typename T>
__global__ void transpose_to_half_kernel(const T* __restrict__ src, __half* __restrict__ dst, int K, int N) {
    // src [K][N] row-major -> dst [N][K] row-major (the K-major layout the tensor core reads)
    __shared__ __half tile[32][33];
    const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int k = k0 + i, n = n0 + threadIdx.x;
        tile[i][threadIdx.x] = (k < K && n < N) ? to_half<T>(src[(size_t)k * N + n]) : __float2half_rn(0.f);
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int n = n0 + i, k = k0 + threadIdx.x;
        if (n < N && k < K) dst[(size_t)n * K + k] = tile[threadIdx.x][i];
    }
}

__global__ void enc_kv_scatter_kernel(const __half* __restrict__ y, __half* kc, __half* vc, int rows_total, int E_dims,
                                      int S, int H, int dh, int dhp) {
    // y [rows_total][2S] -> K, V caches [b][h][e][dh_pad]
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)rows_total * 2 * S) return;
    const int r = (int)(i / (2 * S)), cidx = (int)(i % (2 * S));
    const int b = r / E_dims, e = r % E_dims;
    const int which = cidx / S, cs = cidx % S;
    const int h = cs / dh, d = cs % dh;
    __half* dst = which ? vc : kc;
    dst[(((size_t)(b * H + h)) * E_dims + e) * dhp + d] = y[i];
}

}  // namespace

// =========================================================================================
// host side
// =========================================================================================
namespace {

struct Layout {
    size_t off_dev, off_cols, off_goff, off_lrow, off_streams, off_small, off_cache, off_h, off_x1, off_qkv, off_a, off_g, off_xp[4], off_part, off_prof, off_prof2, off_prof3, off_lnacc, off_encx, off_ency, off_wt, off_pf, off_step, total;
    int KS, U;
    size_t wt_per_layer;
    int pf_len, pf_rows;
    size_t stream_stride;
    std::vector<ushort2> cols;
    std::vector<uint32_t> goff;
    std::vector<int> lrow;
    int lg_on, lg_np;                   // logits GEMM planned, in lg_np passes: its column groups / stream offsets close `cols` / `goff`
    std::vector<size_t> cache_off;      // per layer (K); V follows
    std::vector<size_t> cache_bytes;
    std::vector<int> cache_rows;
    size_t small_per_layer;
    int dh, dh_pad, bc, prime_pad, uni_bytes, kvpre_bytes, nslot, smem_bytes, RC;
    int R;                              // activation rows of the largest kernel this engine launches (16 or 32)
};

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int compute_layout(const jk_prior_config& c, int G, Layout& L) {
    JK_REQUIRE(c.depth >= 1 && c.depth <= JK_MAX_DEPTH, "depth %d out of range", c.depth);
    JK_REQUIRE(c.max_batch >= 1 && c.max_batch <= JK_MAX_BATCH, "max_batch %d out of range (<= %d)", c.max_batch, JK_MAX_BATCH);
    JK_REQUIRE(c.width % 16 == 0 && c.n_state % 16 == 0 && c.mlp_width % 16 == 0,
               "width/n_state/mlp_width must be multiples of 16 (got %d/%d/%d)", c.width, c.n_state, c.mlp_width);
    JK_REQUIRE(c.n_state % c.heads == 0, "n_state %% heads != 0");
    L.dh = c.n_state / c.heads;
    L.dh_pad = head_dim_pad(c);              // MMA k-steps / output pairs of 16 dims
    JK_REQUIRE(L.dh_pad <= 512, "head_dim %d > 512 unsupported", L.dh);
    L.bc = block_len(c);
    JK_REQUIRE(c.blocks == 0 || c.n_ctx % c.blocks == 0, "n_ctx %% blocks != 0");
    L.prime_pad = prime_pad_len(c);
    JK_REQUIRE(L.dh % 2 == 0, "head_dim %d must be even", L.dh);
    const int depth = c.depth;
    // K-split factor: CTAs form units of KS that share column groups and split K.  The largest of 4 / 2 / 1 for which
    // every Conv1D's K splits into whole 16-row MMA steps and no unit gets more than 8 column groups.
    {
        int want = 4;
        if (const char* e = getenv("JK_KSPLIT")) want = atoi(e);
        const int Ks_all[3] = {c.width, c.n_state, c.mlp_width};
        const int Nmax = std::max(std::max(3 * c.n_state, c.width), c.mlp_width);
        int ks = 1;
        for (int cand = 4; cand >= 1; cand >>= 1) {
            if (cand > want || G % cand) continue;
            bool ok = true;
            for (int i = 0; i < 3; ++i) ok = ok && ((Ks_all[i] / 16) % cand == 0);
            ok = ok && ((Nmax / 8 + G / cand - 1) / (G / cand) <= 8);
            if (ok) { ks = cand; break; }
        }
        L.KS = ks; L.U = G / ks;
    }
    const int KS = L.KS, U = L.U;
    // Row count of the shared-memory layout: the 32-row kernel's when more than 16 samples may come.  The K split, the
    // column plan and the streams do not depend on it.
    L.R = c.max_batch > 16 ? 32 : 16;
    const int R = L.R;
    L.cols.assign((size_t)U * depth * 4, make_ushort2(0, 0));
    L.goff.assign((size_t)G * depth * 4, 0);
    std::vector<unsigned long long> cum(U, 0);        // bytes per CTA of a unit (all ranks of a unit stream the same amount)
    std::vector<int> order(U);
    for (int l = 0; l < depth; ++l) {
        const int af = c.attn_func[l];
        JK_REQUIRE(af == 0 || af == 1 || af == 2 || af == 3 || af == 6 || af == 7, "attn_func %d has no decode path", af);
        JK_REQUIRE(af == 0 || c.blocks > 0 || af == 6, "attn_func %d needs blocks", af);
        const int Ks[4] = {c.width, c.n_state, c.width, c.mlp_width};
        const int Ns[4] = {af == 6 ? c.n_state : 3 * c.n_state, c.width, c.mlp_width, c.width};
        for (int gi = 0; gi < 4; ++gi) {
            JK_REQUIRE(Ns[gi] % 8 == 0, "n_out %d not a multiple of 8", Ns[gi]);
            const int groups = Ns[gi] / 8, base = groups / U, extra = groups % U;
            JK_REQUIRE(base + (extra ? 1 : 0) <= 8, "n_out %d too wide for %d units (max 64 columns per unit)", Ns[gi], U);
            std::vector<int> n(U, base);
            if (gi == 1 || gi == 3) {
                // width-W outputs (proj, proj2, and the embedding): ONE fixed assignment for the whole stack, because the
                // CTA that finishes a column keeps that column of the residual stream in its shared memory
                for (int i = 0; i < extra; ++i) n[i] += 1;
            } else {
                // water-filling: each extra group goes to the unit whose stream is shortest so far, a unit may take more
                // than one.  With 33 units (132 SMs, KS = 4) the fixed width-W assignment above leaves 8 units 10 KB per
                // layer behind, more than one extra group per Conv1D can make up: the longest stream of 1b_lyrics was 3.1 %
                // above the shortest, now 0.1 % (tests/test_decode_plan_cpu.py).  Its effect on the step time has not been
                // measured separately.
                const unsigned long long chunk = (unsigned long long)(Ks[gi] / KS / 16) * 256ull;
                for (int i = 0; i < extra; ++i) {
                    int best = -1;
                    for (int u = 0; u < U; ++u)
                        if (n[u] < 8 && (best < 0 || cum[u] + n[u] * chunk < cum[best] + n[best] * chunk)) best = u;
                    n[best] += 1;
                }
            }
            int g0 = 0;
            for (int u = 0; u < U; ++u) {
                L.cols[((size_t)u * depth + l) * 4 + gi] = make_ushort2((unsigned short)g0, (unsigned short)n[u]);
                for (int r = 0; r < KS; ++r)
                    L.goff[((size_t)(u * KS + r) * depth + l) * 4 + gi] = (uint32_t)(cum[u] / 16);
                cum[u] += (unsigned long long)n[u] * (Ks[gi] / KS / 16) * 256ull;
                g0 += n[u];
            }
        }
    }
    // logits GEMM (fifth Conv1D, K' = 2 * width: hi and lo fp16 halves of the fp32 x_out): planned when the K-split is even
    // (a rank's K slice must not straddle the hi / lo boundary) and its [R][2 * width / KS + 8] fp16 tile fits in what the
    // shared-memory union region holds anyway: 64 KB at 16 rows, the 88 KB of the cross-warp reduction at 32.  A unit
    // multiplies at most 8 column groups per pass (the partial-sum exchange holds 64 columns); wider vocabularies take more
    // passes, each with its own exchange buffer, so at most 4 (1b_lyrics on 132 SMs: 266 groups over 33 units, 2 passes).
    // Its records are appended to `cols` ([passes][U] entries) and `goff` ([passes][G] entries), pass after pass.
    L.lg_on = 0; L.lg_np = 0;
    {
        const int groups = (c.bins + 7) / 8;           // a ragged last group is padded with zero weights
        const int Kp = 2 * c.width;
        const int np = ((groups + U - 1) / U + 7) / 8;
        const size_t tile_cap = std::max((size_t)65536, (size_t)red_bytes(R) + 2 * 1024 * 8);
        const bool ok = c.bins > 0 && KS >= 2 && (Kp / 16) % KS == 0 && c.width % (Kp / KS) == 0 &&
                        (size_t)R * (Kp / KS + 8) * 2 <= tile_cap && np <= 4 && !getenv("JK_NO_LOGITS_MMA");
        if (ok) {
            L.lg_on = 1; L.lg_np = np;
            L.cols.resize((size_t)U * depth * 4 + (size_t)np * U, make_ushort2(0, 0));
            L.goff.resize((size_t)G * depth * 4 + (size_t)np * G, 0);
            const int base = groups / U, extra = groups % U;
            std::vector<int> n(U, base);
            for (int i = 0; i < U; ++i) order[i] = i;
            std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cum[a] < cum[b]; });
            for (int i = 0; i < extra; ++i) n[order[i]] += 1;
            // pass p of unit u: the next min(8, rest) groups of the unit's contiguous range
            std::vector<int> g0(U, 0);
            for (int u = 1; u < U; ++u) g0[u] = g0[u - 1] + n[u - 1];
            for (int p = 0; p < np; ++p) {
                for (int u = 0; u < U; ++u) {
                    const int k = std::max(0, std::min(8, n[u] - 8 * p));
                    L.cols[(size_t)U * depth * 4 + (size_t)p * U + u] = make_ushort2((unsigned short)(g0[u] + 8 * p), (unsigned short)k);
                    for (int r = 0; r < KS; ++r) L.goff[(size_t)G * depth * 4 + (size_t)p * G + u * KS + r] = (uint32_t)(cum[u] / 16);
                    cum[u] += (unsigned long long)k * (Kp / KS / 16) * 256ull;
                }
            }
        }
    }
    unsigned long long mx = 0;
    for (int u = 0; u < U; ++u) mx = std::max(mx, cum[u]);
    JK_REQUIRE(mx / 16 < 0xffffffffull, "stream too long");
    L.stream_stride = align_up((size_t)mx + 256, 256);
    L.lrow.assign(G + 1, 0);
    for (int cta = 0; cta <= G; ++cta) L.lrow[cta] = (int)((long long)c.bins * cta / G);

    const int Kmax = std::max(c.width, std::max(c.n_state, c.mlp_width)) / KS;
    // rows >= n_samples of the A tile are never read back (see stage_acts)
    const int act_rows = R == 32 ? 32 : c.max_batch > 8 ? 16 : 8;
    const int max_smem = 232448;
    int RC = attn_tile_rows(L.dh_pad), nslot = 0;
    for (;; RC >>= 1) {
        size_t uni = (size_t)act_rows * (Kmax + 8) * 2;
        uni = std::max(uni, (size_t)R * logit_kt(R) * 4);    // fp32 logits y tile (64 KB)
        if (L.lg_on) uni = std::max(uni, (size_t)R * (2 * c.width / KS + 8) * 2);     // the logits GEMM's A tile
        uni = std::max(uni, (size_t)red_bytes(R) + 2 * 1024 * 8);                     // cross-warp reduction + statistics scratch
        const size_t kv_stage = (size_t)2 * RC * L.dh_pad * 2;                        // one K tile + one V tile
        size_t attn = kv_stage + (size_t)3 * L.dh_pad * 2 + 64 * 4 + (size_t)L.dh_pad * 4 + 64;   // tiles, q/k/v, scores, running output
        uni = std::max(uni, attn);
        L.uni_bytes = (int)align_up(uni, 1024);
        L.kvpre_bytes = (int)align_up(kv_stage, 1024);      // second K/V stage (double buffer of multi-tile parts)
        nslot = (max_smem - kHeaderBytes - L.uni_bytes - L.kvpre_bytes) / kSlotBytes;
        if (nslot >= 4 || RC <= 16) break;                  // a deep weight ring matters more than tall K/V tiles
    }
    L.RC = RC;
    nslot = std::min(nslot, kMaxSlots);
    // More than 16 samples take the 32-row kernel, whose whole [32][K / KS + 8] activation tile must sit in shared memory
    // next to the K/V tiles and at least 4 ring slots (5b_lyrics: K split 1, 308 KB).
    JK_REQUIRE(R == 16 || nslot >= 4,
               "max_batch %d > 16 needs a [32 x %d] fp16 activation tile (%zu bytes: K %d, K split %d) in the %d bytes of "
               "shared memory per CTA, which leaves %d weight-ring slots (at least 4); this configuration takes at most 16 samples",
               c.max_batch, Kmax + 8, (size_t)32 * (Kmax + 8) * 2, Kmax * KS, KS, max_smem, std::max(nslot, 0));
    JK_REQUIRE(nslot >= 2, "not enough shared memory for the weight ring (uni %d bytes)", L.uni_bytes);
    L.nslot = nslot;
    L.smem_bytes = kHeaderBytes + L.uni_bytes + L.kvpre_bytes + nslot * kSlotBytes;
    // ldmatrix always addresses 16 A-tile rows; with an 8-row tile rows 8..15 must still lie inside the allocation
    JK_REQUIRE((size_t)kHeaderBytes + (size_t)std::max(16, act_rows) * (Kmax + 8) * 2 <= (size_t)L.smem_bytes, "A tile exceeds shared memory");

    size_t off = 0;
    L.off_dev = off; off = align_up(off + sizeof(EngineDev), 256);
    L.off_cols = off; off = align_up(off + L.cols.size() * sizeof(ushort2), 256);
    L.off_goff = off; off = align_up(off + L.goff.size() * 4, 256);
    L.off_lrow = off; off = align_up(off + L.lrow.size() * 4, 256);
    L.off_streams = off; off = align_up(off + (size_t)G * L.stream_stride, 256);
    // per layer small params: 4 biases + 4 LN vectors (+ enc kv weights/bias for type 6)
    L.small_per_layer = align_up((size_t)(3 * c.n_state + c.width + c.mlp_width + c.width + 4 * c.width) * 4, 256);
    L.off_small = off; off += L.small_per_layer * depth;
    for (int l = 0; l < depth; ++l)
        if (c.attn_func[l] == 6) off = align_up(off + (size_t)c.width * 2 * c.n_state * 2 + 2 * c.n_state * 4 + 512, 256);
    L.off_cache = off;
    L.cache_off.resize(depth); L.cache_bytes.resize(depth); L.cache_rows.resize(depth);
    for (int l = 0; l < depth; ++l) {
        int rows = cache_rows_for(c, c.attn_func[l], L.bc, L.prime_pad);
        L.cache_rows[l] = rows;
        size_t bytes = align_up((size_t)c.max_batch * c.heads * rows * L.dh_pad * 2, 256);
        L.cache_off[l] = off; L.cache_bytes[l] = bytes;
        off += 2 * bytes;
    }
    // LL activation buffers: 8 bytes per fp16 PAIR ({half2, flag})
    L.off_h = off;   off = align_up(off + (size_t)R * c.width * 4, 256);
    L.off_x1 = off;  off = align_up(off + (size_t)R * c.width * 4, 256);
    L.off_qkv = off; off = align_up(off + (size_t)R * 3 * c.n_state * 4, 256);
    L.off_a = off;   off = align_up(off + (size_t)R * c.n_state * 4, 256);
    L.off_g = off;   off = align_up(off + (size_t)R * c.mlp_width * 4, 256);
    for (int gi = 0; gi < 4; ++gi) { L.off_xp[gi] = off; off = align_up(off + (size_t)G * R * kXpCols * 8, 256); }
    L.off_part = off; off = align_up(off + (size_t)c.max_batch * c.heads * kMaxSplit * (L.dh_pad + 2) * 8, 256);      // LL words
    L.off_prof = off; off = align_up(off + (size_t)kProfSlots * 8, 256);
    L.off_prof2 = off; off = align_up(off + (size_t)kProfSlots * 8 * 8, 256);
    L.off_prof3 = off; off = align_up(off + (size_t)5 * 256 * 2 * 8, 256);
    L.off_lnacc = off; off = align_up(off + (size_t)(2 * depth + 1) * 512 * 8, 256);
    {
        bool any6 = false;
        for (int l = 0; l < depth; ++l) any6 = any6 || (c.attn_func[l] == 6);
        L.off_encx = off; if (any6) off = align_up(off + (size_t)c.max_batch * c.encoder_dims * c.width * 2, 1024);
        L.off_ency = off; if (any6) off = align_up(off + (size_t)c.max_batch * c.encoder_dims * 2 * c.n_state * 2, 1024);
    }
    {   // chunked prefill: K-major fp16 weight copies + activation workspace (prefill.cu).  Every GEMM K must give
        // 16-byte rows (K % 8) and fill at least one GEMM K block; K tails are zero-filled by TMA.  The workspace
        // holds a whole window (n_ctx positions x max_batch: 2.8 GB for 1b_lyrics of the H100's 80 GB),
        // so continuation windows re-prime their 4096 given tokens in one pass; JK_PREFILL_MAX lowers it.
        auto k_ok = [](int k) { return k >= 64 && k % 8 == 0; };
        const bool ok = k_ok(c.width) && k_ok(c.n_state) && k_ok(c.mlp_width) && !getenv("JK_NO_PREFILL");
        int cap = c.n_ctx;
        if (const char* e = getenv("JK_PREFILL_MAX")) cap = std::max(2, std::min(cap, atoi(e)));
        L.pf_len = ok ? cap : 0;
        L.pf_rows = c.max_batch * L.pf_len;
        L.wt_per_layer = align_up((size_t)(3 * c.n_state * c.width + c.width * c.n_state + 2 * c.mlp_width * c.width) * 2, 1024);
        L.off_wt = off; if (ok) off = align_up(off + L.wt_per_layer * depth, 1024);
        L.off_pf = off;
        if (ok) off = align_up(off + (size_t)L.pf_rows * (3 * c.width + 3 * c.n_state + c.n_state + c.mlp_width) * 2, 1024);
    }
    L.off_step = off; off += 256;                       // step count and position, one 128-byte line each
    L.total = off;
    return 0;
}

int device_sms() {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return sms;
}

}  // namespace

extern "C" int jk_device_sm_count(int* out) {
    int s = device_sms();
    JK_REQUIRE(s > 0, "no CUDA device");
    *out = s;
    return 0;
}

extern "C" int jk_prior_arena_bytes(const jk_prior_config* cfg, size_t* bytes) {
    JK_REQUIRE(cfg && bytes, "null argument");
    int G = device_sms();
    JK_REQUIRE(G > 0, "no CUDA device (the decode engine has no CPU path)");
    Layout L;
    int rc = compute_layout(*cfg, G, L);
    if (rc) return rc;
    *bytes = L.total;
    return 0;
}

extern "C" int jk_prior_config_prefill_capacity(const jk_prior_config* cfg, int* max_positions) {
    JK_REQUIRE(cfg && max_positions, "null argument");
    int G = device_sms();
    JK_REQUIRE(G > 0, "no CUDA device (the decode engine has no CPU path)");
    Layout L;
    int rc = compute_layout(*cfg, G, L);
    if (rc) return rc;
    *max_positions = L.pf_len;
    return 0;
}

extern "C" int jk_prior_plan(const jk_prior_config* cfg, int n_sms, jk_prior_plan_info* out, uint16_t* cols, size_t cols_len) {
    JK_REQUIRE(cfg && out, "null argument");
    JK_REQUIRE(n_sms >= 1 && n_sms <= 1024, "n_sms %d out of range", n_sms);
    Layout L;
    int rc = compute_layout(*cfg, n_sms, L);
    if (rc) return rc;
    out->k_split = L.KS; out->units = L.U; out->ring_slots = L.nslot; out->smem_bytes = L.smem_bytes; out->tile_rows = L.RC;
    out->logits_passes = L.lg_np;
    out->arena_bytes = (uint64_t)L.total; out->stream_stride = (uint64_t)L.stream_stride;
    if (cols) {
        const size_t ncols = L.cols.size();                       // the layers' records, then the logits GEMM's
        JK_REQUIRE(cols_len >= ncols * 2, "cols buffer too small: %zu < %zu", cols_len, ncols * 2);
        for (size_t i = 0; i < ncols; ++i) { cols[2 * i] = L.cols[i].x; cols[2 * i + 1] = L.cols[i].y; }
    }
    return 0;
}

extern "C" int jk_prior_create(const jk_prior_config* cfg, void* arena, size_t arena_bytes, jk_prior** out,
                               jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(cfg && arena && out, "null argument");
    int G = device_sms();
    JK_REQUIRE(G > 0, "no CUDA device (the decode engine has no CPU path)");
    Layout L;
    int rc = compute_layout(*cfg, G, L);
    if (rc) return rc;
    JK_REQUIRE(arena_bytes >= L.total, "arena too small: %zu < %zu", arena_bytes, L.total);
    JK_REQUIRE(((uintptr_t)arena & 255) == 0, "arena must be 256-byte aligned");
    JK_CHECK_CUDA(cudaMemsetAsync(arena, 0, L.total, stream));
    jk_prior* p = new jk_prior();
    p->cfg = *cfg; p->arena = (uint8_t*)arena; p->arena_bytes = arena_bytes; p->G = G; p->t_host = 0;
    p->smem_bytes = L.smem_bytes;
    p->cols = L.cols; p->goff = L.goff;
    if (getenv("JK_VERBOSE"))
        fprintf(stderr, "jk_prior_create: G %d, KS %d, units %d, tile rows %d, ring %d x %d B, uni %d B, smem %d B, arena %.1f MB\n", G, L.KS,
                L.U, L.RC, L.nslot, kSlotBytes, L.uni_bytes, L.smem_bytes, L.total / 1e6);
    uint8_t* A = p->arena;
    EngineDev& E = p->host;
    memset(&E, 0, sizeof(E));
    E.W = cfg->width; E.S = cfg->n_state; E.M = cfg->mlp_width; E.H = cfg->heads; E.dh = L.dh; E.dh_pad = L.dh_pad;
    E.L = cfg->n_ctx; E.blocks = cfg->blocks; E.bc = L.bc; E.bins = cfg->bins; E.prime_pad = L.prime_pad;
    E.enc_dims = cfg->encoder_dims; E.Bmax = cfg->max_batch; E.add_cond_after = cfg->add_cond_after;
    E.depth = cfg->depth; E.G = G; E.KS = L.KS; E.ks_shift = L.KS == 4 ? 2 : L.KS == 2 ? 1 : 0; E.U = L.U; E.RC = L.RC; E.nslot = L.nslot; E.uni_bytes = L.uni_bytes; E.kvpre_bytes = L.kvpre_bytes; E.small_bytes = (int)L.small_per_layer; E.prof_on = getenv("JK_PROFILE") ? 1 : 0;
    {
        const int nowait = getenv("JK_NOWAIT") ? atoi(getenv("JK_NOWAIT")) : 0;
        JK_CHECK_CUDA(cudaMemcpyToSymbol(jk_nowait, &nowait, sizeof(int)));
    }
    E.scale2 = attn_scale2(L.dh);
    E.cols = (const ushort2*)(A + L.off_cols);
    p->d_cols = (ushort2*)(A + L.off_cols);
    p->d_goff = (uint32_t*)(A + L.off_goff);
    E.lrow0 = (const int*)(A + L.off_lrow);
    E.lg_on = L.lg_on; p->lg_on = L.lg_on;
    E.lg_np = L.lg_np; p->lg_np = L.lg_np;
    E.lg_cols = (const ushort2*)(A + L.off_cols) + (size_t)L.U * cfg->depth * 4;
    E.lg_goff = (const uint32_t*)(A + L.off_goff) + (size_t)G * cfg->depth * 4;
    E.streams = A + L.off_streams; E.stream_stride = L.stream_stride;
    E.ll_h = (unsigned long long*)(A + L.off_h); E.ll_x1 = (unsigned long long*)(A + L.off_x1);
    E.ll_qkv = (unsigned long long*)(A + L.off_qkv); E.ll_a = (unsigned long long*)(A + L.off_a);
    E.ll_g = (unsigned long long*)(A + L.off_g);
    for (int gi = 0; gi < 4; ++gi) E.xp[gi] = (unsigned long long*)(A + L.off_xp[gi]);
    E.part = (unsigned long long*)(A + L.off_part);
    E.prof = (unsigned long long*)(A + L.off_prof);
    E.lnacc = (long long*)(A + L.off_lnacc);
    E.prof2 = (long long*)(A + L.off_prof2);
    E.prof3 = (unsigned long long*)(A + L.off_prof3);
    E.step = (unsigned*)(A + L.off_step); E.t = (int*)(A + L.off_step + 128);
    size_t enc_off = L.off_small + L.small_per_layer * cfg->depth;
    for (int i = 0; i < 4; ++i) { p->bias_ptr[i].resize(cfg->depth); p->ln_ptr[i].resize(cfg->depth); }
    p->enc_w.assign(cfg->depth, nullptr); p->enc_b.assign(cfg->depth, nullptr);
    for (int l = 0; l < cfg->depth; ++l) {
        LayerDev& LD = E.layer[l];
        LD.attn_func = cfg->attn_func[l];
        LD.rows = L.cache_rows[l];
        LD.kc = (__half*)(A + L.cache_off[l]);
        LD.vc = (__half*)(A + L.cache_off[l] + L.cache_bytes[l]);
        float* s = (float*)(A + L.off_small + L.small_per_layer * l);
        p->bias_ptr[0][l] = s; s += 3 * cfg->n_state;
        p->bias_ptr[1][l] = s; s += cfg->width;
        p->bias_ptr[2][l] = s; s += cfg->mlp_width;
        p->bias_ptr[3][l] = s; s += cfg->width;
        for (int i = 0; i < 4; ++i) { p->ln_ptr[i][l] = s; s += cfg->width; }
        LD.b_qkv = p->bias_ptr[0][l]; LD.b_o = p->bias_ptr[1][l]; LD.b_1 = p->bias_ptr[2][l]; LD.b_2 = p->bias_ptr[3][l];
        LD.ln0_g = p->ln_ptr[0][l]; LD.ln0_b = p->ln_ptr[1][l]; LD.ln1_g = p->ln_ptr[2][l]; LD.ln1_b = p->ln_ptr[3][l];
        if (cfg->attn_func[l] == 6) {
            p->enc_w[l] = (__half*)(A + enc_off);
            p->enc_b[l] = (float*)(A + enc_off + (size_t)cfg->width * 2 * cfg->n_state * 2);
            enc_off = align_up(enc_off + (size_t)cfg->width * 2 * cfg->n_state * 2 + 2 * cfg->n_state * 4 + 512, 256);
            LD.enc_w = p->enc_w[l]; LD.enc_b = p->enc_b[l];
        }
    }
    p->enc_x16 = (__half*)(A + L.off_encx); p->enc_y16 = (__half*)(A + L.off_ency);
    p->pf_rows = L.pf_rows; p->pf_len = L.pf_len;
    for (int i = 0; i < 4; ++i) p->wt[i].assign(cfg->depth, nullptr);
    if (L.pf_rows) {
        for (int l = 0; l < cfg->depth; ++l) {
            __half* w = (__half*)(A + L.off_wt + L.wt_per_layer * l);
            p->wt[0][l] = w; w += (size_t)3 * cfg->n_state * cfg->width;
            p->wt[1][l] = w; w += (size_t)cfg->width * cfg->n_state;
            p->wt[2][l] = w; w += (size_t)cfg->mlp_width * cfg->width;
            p->wt[3][l] = w;
        }
        __half* a = (__half*)(A + L.off_pf);
        const size_t R = (size_t)L.pf_rows;
        p->pf_x = a; a += R * cfg->width;
        p->pf_xn = a; a += R * cfg->width;
        p->pf_x1 = a; a += R * cfg->width;
        p->pf_qkv = a; a += R * 3 * cfg->n_state;
        p->pf_a = a; a += R * cfg->n_state;
        p->pf_g = a;
    }
    p->dev = (EngineDev*)(A + L.off_dev);
    JK_CHECK_CUDA(cudaMemcpyAsync(A + L.off_cols, L.cols.data(), L.cols.size() * sizeof(ushort2), cudaMemcpyHostToDevice, stream));
    JK_CHECK_CUDA(cudaMemcpyAsync(A + L.off_goff, L.goff.data(), L.goff.size() * 4, cudaMemcpyHostToDevice, stream));
    JK_CHECK_CUDA(cudaMemcpyAsync(A + L.off_lrow, L.lrow.data(), L.lrow.size() * 4, cudaMemcpyHostToDevice, stream));
    JK_CHECK_CUDA(cudaMemcpyAsync(p->dev, &p->host, sizeof(EngineDev), cudaMemcpyHostToDevice, stream));
    JK_CHECK_CUDA(cudaStreamSynchronize(stream));      // the host vectors above go out of scope
    {   // the attribute belongs to the KERNEL, not to this engine: engines of different configurations coexist
        // (5b_lyrics: lyric encoder + decoder), so it is raised to the device's opt-in maximum once and never lowered
        int dev = 0, optin = 0;
        JK_CHECK_CUDA(cudaGetDevice(&dev));
        JK_CHECK_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        JK_REQUIRE(L.smem_bytes <= optin, "decode kernel needs %d bytes of shared memory, device allows %d", L.smem_bytes, optin);
        JK_CHECK_CUDA(cudaFuncSetAttribute(jk_decode_step_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
        JK_CHECK_CUDA(cudaFuncSetAttribute(jk_decode_step_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin));
    }
    *out = p;
    return 0;
}

extern "C" int jk_prior_destroy(jk_prior* p) {
    delete p;
    return 0;
}

template <typename T>
static int pack_one(jk_prior* p, const void* w, int K, int N, int l, int gi, cudaStream_t stream) {
    pack_gemm_kernel<T><<<p->G, 256, 0, stream>>>((const T*)w, K, N, (uint8_t*)p->host.streams, p->host.stream_stride,
                                                   p->d_cols, p->d_goff, p->cfg.depth, l, gi, p->host.KS);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}
template <typename T>
static int round_bias(const void* src, float* dst, int n, cudaStream_t stream) {
    round_bias_kernel<T><<<(n + 255) / 256, 256, 0, stream>>>((const T*)src, dst, n);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int jk_prior_load_layer(jk_prior* p, int l, const jk_layer_weights* w, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(p && w, "null argument");
    JK_REQUIRE(l >= 0 && l < p->cfg.depth, "layer %d out of range", l);
    const jk_prior_config& c = p->cfg;
    const int af = c.attn_func[l];
    const int Ks[4] = {c.width, c.n_state, c.width, c.mlp_width};
    const int Ns[4] = {af == 6 ? c.n_state : 3 * c.n_state, c.width, c.mlp_width, c.width};
    const void* ws[4] = {w->c_attn_w, w->c_proj_w, w->fc_w, w->proj2_w};
    const void* bs[4] = {w->c_attn_b, w->c_proj_b, w->fc_b, w->proj2_b};
    for (int gi = 0; gi < 4; ++gi) {
        JK_REQUIRE(ws[gi] && bs[gi], "layer %d: missing weight %d", l, gi);
        int rc = w->w_dtype ? pack_one<__half>(p, ws[gi], Ks[gi], Ns[gi], l, gi, stream)
                            : pack_one<float>(p, ws[gi], Ks[gi], Ns[gi], l, gi, stream);
        if (rc) return rc;
        rc = w->b_dtype ? round_bias<__half>(bs[gi], p->bias_ptr[gi][l], Ns[gi], stream)
                        : round_bias<float>(bs[gi], p->bias_ptr[gi][l], Ns[gi], stream);
        if (rc) return rc;
    }
    if (p->pf_rows) {      // K-major fp16 copies for the tensor-core prefill
        for (int gi = 0; gi < 4; ++gi) {
            dim3 tg((Ns[gi] + 31) / 32, (Ks[gi] + 31) / 32), tb(32, 8);
            if (w->w_dtype) transpose_to_half_kernel<__half><<<tg, tb, 0, stream>>>((const __half*)ws[gi], p->wt[gi][l], Ks[gi], Ns[gi]);
            else transpose_to_half_kernel<float><<<tg, tb, 0, stream>>>((const float*)ws[gi], p->wt[gi][l], Ks[gi], Ns[gi]);
            JK_CHECK_CUDA(cudaGetLastError());
        }
    }
    const float* lns[4] = {w->ln0_g, w->ln0_b, w->ln1_g, w->ln1_b};
    for (int i = 0; i < 4; ++i) {
        JK_REQUIRE(lns[i], "layer %d: missing LayerNorm parameter %d", l, i);
        JK_CHECK_CUDA(cudaMemcpyAsync(p->ln_ptr[i][l], lns[i], (size_t)c.width * 4, cudaMemcpyDeviceToDevice, stream));
    }
    if (af == 6) {
        JK_REQUIRE(w->c_enc_kv_w && w->c_enc_kv_b, "layer %d: attn_func 6 needs c_enc_kv", l);
        dim3 tg((2 * c.n_state + 31) / 32, (c.width + 31) / 32), tb(32, 8);
        if (w->w_dtype) transpose_to_half_kernel<__half><<<tg, tb, 0, stream>>>((const __half*)w->c_enc_kv_w, p->enc_w[l], c.width, 2 * c.n_state);
        else transpose_to_half_kernel<float><<<tg, tb, 0, stream>>>((const float*)w->c_enc_kv_w, p->enc_w[l], c.width, 2 * c.n_state);
        JK_CHECK_CUDA(cudaGetLastError());
        int rc = w->b_dtype ? round_bias<__half>(w->c_enc_kv_b, p->enc_b[l], 2 * c.n_state, stream)
                            : round_bias<float>(w->c_enc_kv_b, p->enc_b[l], 2 * c.n_state, stream);
        if (rc) return rc;
    }
    return 0;
}

extern "C" int jk_prior_set_embeddings(jk_prior* p, const float* x_emb, const float* pos_emb, const float* x_out,
                                       const float* start_token) {
    JK_REQUIRE(p, "null engine");
    p->host.x_emb = x_emb; p->host.pos_emb = pos_emb; p->host.x_out = x_out; p->host.start_token = start_token;
    JK_CHECK_CUDA(cudaMemcpy(p->dev, &p->host, sizeof(EngineDev), cudaMemcpyHostToDevice));
    if (p->lg_on && x_out) {       // logits GEMM: hi / lo fp16 fragment streams of x_out, behind every CTA's last layer
        pack_logits_kernel<<<dim3(p->G, p->lg_np), 256>>>(x_out, p->cfg.width, p->cfg.bins, (uint8_t*)p->host.streams, p->host.stream_stride,
                                          p->host.lg_cols, p->host.lg_goff, p->host.KS);
        JK_CHECK_CUDA(cudaGetLastError());
        JK_CHECK_CUDA(cudaDeviceSynchronize());
    }
    return 0;
}

extern "C" int jk_prior_reset(jk_prior* p, int t0, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(p, "null engine");
    JK_REQUIRE(t0 >= 0 && t0 <= p->cfg.n_ctx, "t0 out of range");
    JK_CHECK_CUDA(cudaMemcpyAsync(p->host.t, &t0, sizeof(int), cudaMemcpyHostToDevice, stream));
    JK_CHECK_CUDA(cudaStreamSynchronize(stream));
    p->t_host = t0;
    return 0;
}

extern "C" int jk_prior_set_encoder_kv(jk_prior* p, const float* encoder_kv, int n, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(p && encoder_kv, "null argument");
    const jk_prior_config& c = p->cfg;
    JK_REQUIRE(n >= 1 && n <= c.max_batch, "n_samples out of range");
    const int rows = n * c.encoder_dims;
    JK_REQUIRE(c.width >= 64 && c.width % 8 == 0, "encoder-decoder layers need width >= 64 and width %% 8 == 0 (GEMM operand rows)");
    {   // encoder_kv.type_as(x): fp32 -> fp16 once, shared by every enc-dec layer
        const size_t cnt = (size_t)rows * c.width;
        to_half_kernel<float><<<(unsigned)((cnt + 255) / 256), 256, 0, stream>>>(encoder_kv, p->enc_x16, cnt);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    for (int l = 0; l < c.depth; ++l) {
        if (c.attn_func[l] != 6) continue;
        int rc = jk_conv1d_prefill_f16(p->enc_x16, p->enc_w[l], p->enc_b[l], p->enc_y16, rows, 2 * c.n_state, c.width, stream_);
        if (rc) return rc;
        const size_t cnt = (size_t)rows * 2 * c.n_state;
        enc_kv_scatter_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, stream>>>(p->enc_y16, p->host.layer[l].kc, p->host.layer[l].vc,
                                                                                  rows, c.encoder_dims, c.n_state, c.heads,
                                                                                  p->host.dh, p->host.dh_pad);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

extern "C" int jk_prior_step(jk_prior* p, const jk_step_args* a, jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(p && a, "null argument");
    JK_REQUIRE(a->n_samples >= 1 && a->n_samples <= p->cfg.max_batch, "n_samples %d out of range (max_batch %d)",
               a->n_samples, p->cfg.max_batch);
    JK_REQUIRE(p->t_host >= 0, "the last prefill stopped early (n_layers) and left later layers' caches unfilled: "
                               "call jk_prior_reset first");
    JK_REQUIRE(p->t_host < p->cfg.n_ctx, "position %d is past the context (n_ctx %d): reset the engine", p->t_host, p->cfg.n_ctx);
    JK_REQUIRE(a->x_in || a->tokens || p->t_host == 0, "tokens required for t > 0");
    JK_REQUIRE(a->x_in || (p->host.pos_emb && p->host.x_emb), "embeddings not set (jk_prior_set_embeddings)");
    JK_REQUIRE(!a->logits || p->host.x_out, "x_out not set");
    JK_REQUIRE(a->x_cond_len == 0 || a->x_cond_len == 1 || a->x_cond_len == p->cfg.n_ctx, "x_cond_len must be 1 or n_ctx");
    StepArgs A;
    A.n = a->n_samples; A.x_in = a->x_in; A.tokens = (const long long*)a->tokens; A.tok_stride = a->tok_stride;
    A.y_cond = a->y_cond; A.x_cond = a->x_cond; A.x_cond_len = a->x_cond_len ? a->x_cond_len : 1;
    A.h_out = a->h_out; A.logits = a->logits; A.logits_bstride = a->logits_bstride; A.logits_tstride = a->logits_tstride;
    A.logit_bias = a->logit_bias; A.lb_bstride = a->logit_bias_bstride; A.lb_tstride = a->logit_bias_tstride;
    const EngineDev* E = p->dev;
    void* args[2] = {(void*)&E, (void*)&A};
    // Up to 16 samples take the 16-row kernel even on an engine planned for 32: its layout holds the 16-row one, and one
    // m16 tile per weight fragment is all those rows need.
    const void* kernel = a->n_samples <= 16 ? (const void*)jk_decode_step_kernel<16> : (const void*)jk_decode_step_kernel<32>;
    JK_CHECK_CUDA(cudaLaunchCooperativeKernel(kernel, dim3(p->G), dim3(kThreads), args, (size_t)p->smem_bytes, stream));
    p->t_host += 1;
    return 0;
}

extern "C" int jk_prior_has_logits_gemm(const jk_prior* p, int* on) {
    JK_REQUIRE(p && on, "null argument");
    *on = p->lg_on ? 1 : 0;
    return 0;
}

extern "C" int jk_prior_position(const jk_prior* p, int* t) {
    JK_REQUIRE(p && t, "null argument");
    *t = p->t_host;
    return 0;
}

extern "C" int jk_prior_debug_buffer(const jk_prior* p, int which, const void** ptr, size_t* n) {
    JK_REQUIRE(p && ptr && n, "null argument");
    const jk_prior_config& c = p->cfg;
    switch (which) {
        /* 0..4 were the fp16 intermediates of round 1; activations now travel as LL words between SMs */
        case 5: *ptr = p->host.prof; *n = (size_t)kProfSlots * 4; break;     /* uint64 timestamps */
        case 7: *ptr = p->host.prof3; *n = (size_t)5 * 256 * 2 * 4; break;
        case 6: *ptr = p->host.prof2; *n = (size_t)kProfSlots * 8 * 4; break; /* int64 clock64 stamps [slot][8] */
        default: JK_REQUIRE(false, "unknown buffer %d", which);
    }
    return 0;
}
