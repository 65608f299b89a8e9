// Engine descriptor shared by the decode kernel (decode_engine.cu) and the chunked prefill (prefill.cu).
#pragma once
#include "common.cuh"
#include "../../include/jkb200.h"
#include <vector>

namespace jk {

struct LayerDev {
    int attn_func;
    int rows;                       // cache rows per (b, h)
    __half* kc;
    __half* vc;                     // [B][H][rows][dh_pad]
    const float *ln0_g, *ln0_b, *ln1_g, *ln1_b;
    const float *b_qkv, *b_o, *b_1, *b_2;   // fp32 holding fp16-rounded biases
    const __half* enc_w;            // [W][2S] fp16 copy of c_enc_kv.w (attn_func 6)
    const float* enc_b;
};

struct EngineDev {
    int W, S, M, H, dh, dh_pad, L, blocks, bc, bins, prime_pad, enc_dims, Bmax, add_cond_after, depth, G;
    int RC;                         // rows of one shared-memory K (or V) tile of the attention phase
    int ks_shift;                   // log2(KS)
    int KS, U;                      // K-split factor of every Conv1D and the number of column units (G = U * KS)
    int nslot, uni_bytes, kvpre_bytes, small_bytes, prof_on;
    float scale2;
    const ushort2* cols;            // [U][depth][4] : (first 8-column group, number of groups) of a unit
    const uint8_t* streams;
    unsigned long long stream_stride;
    // activations between phases travel as "LL" words (NCCL's low-latency protocol): 8 bytes = {half2 data, u32 flag},
    // written with one 8-byte store and polled by the consumer - no separate flag, no grid barrier
    unsigned long long *ll_h, *ll_x1, *ll_qkv, *ll_a, *ll_g;   // [R][N/2], R = 32 rows when max_batch > 16, else 16
    unsigned long long* xp[4];      // K-split partial sums {fp32, flag}: [G][R][64] per Conv1D of a layer
    unsigned long long* part;       // split-KV partials as LL words {fp32, flag}: [Bmax*H][kMaxSplit][m, l, dh_pad outputs]
    // LayerNorm statistics: 2*depth+1 blocks of 512 words; row r's fixed-point {sum, sumsq} are words 16r and 16r+1
    // (one 128-B line per row), the contributor count in their top bits.  Block 2l feeds layer l's LN0, 2l+1 its LN1;
    // block 2*depth (the final residual stream) only tells the housekeeping warp that every CTA is through the stack.
    long long* lnacc;
    long long* prof2;               // [kProfSlots][8] intra-phase clock64 stamps of CTA 0 (tuning aid)
    unsigned long long* prof3;      // [5][256][2] per-CTA phase entry / exit times of layer 1
    unsigned long long* prof;       // [kProfSlots] phase timestamps of CTA 0 (globaltimer ns)
    unsigned* step;                 // steps executed so far (flags of the next launch derive from it)
    int* t;                         // position of the next step; on its own 128-B line, apart from `step`
    const float *x_emb, *pos_emb, *x_out, *start_token;
    const int* lrow0;               // [G+1] logits rows per CTA (prefix)
    // logits as a fifth Conv1D on the tensor cores (decode_engine.cu "logits GEMM"): 0 when the configuration keeps
    // the fp32 FMA path.  It runs in lg_np passes of at most 8 column groups per unit (the partial-sum exchange holds 64
    // columns): column groups per unit [lg_np][U] and stream offsets per CTA [lg_np][G] (16-byte units)
    int lg_on, lg_np;
    const ushort2* lg_cols;
    const uint32_t* lg_goff;
    LayerDev layer[JK_MAX_DEPTH];
};

// Geometry of the K / V caches (DESIGN §4), from the configuration alone: compute_layout sizes the caches with it and the
// sample selection (select.cu) plans its copies with it, with or without an engine.
inline int head_dim_pad(const jk_prior_config& c) { return (c.n_state / c.heads + 15) / 16 * 16; }   // MMA k-steps of 16
inline int block_len(const jk_prior_config& c) { return c.blocks > 0 ? c.n_ctx / c.blocks : c.n_ctx; }
inline int prime_pad_len(const jk_prior_config& c) { return c.blocks > 0 ? (c.prime_len / c.blocks + 1) * c.blocks : 0; }
// rows per (sample, head) of a layer's cache: the positions its attention pattern reads, the encoder rows (6) or the
// padded prime (7); -1 for an attn_func without a decode path
inline int cache_rows_for(const jk_prior_config& c, int af, int bc, int prime_pad) {
    switch (af) {
        case 0: return c.n_ctx;
        case 1: return bc;
        case 2: return c.n_ctx;
        case 3: return 2 * bc;
        case 6: return c.encoder_dims;
        case 7: return prime_pad;
    }
    return -1;
}

// the attention scores' scale dh^-1/2, as the reference applies it to q and k in two halves:
// scale = 1/sqrt(sqrt(dh)); w.mul_(scale*scale)  (factored_attention.py:83-88)
inline float attn_scale2(int dh) {
    const double sc = 1.0 / sqrt(sqrt((double)dh));
    return (float)(sc * sc);
}

// prefill_gemm.cu: Y = epi(X . W^T + bias [, res]) on wgmma; w_t is [N, K] fp16.
//   epi 0: fp16(acc + b)   1: fp16(quick_gelu(fp16(acc + b)))   2: fp16(res + fp16(acc + b))
int gemm_f16_tc(const void* x, const void* w_t, const float* bias, const void* res, void* y, int M, int N, int K,
                int epi, cudaStream_t stream);

}  // namespace jk

struct jk_prior {
    jk_prior_config cfg;
    jk::EngineDev host;            // host mirror of the device struct
    jk::EngineDev* dev;            // in arena
    uint8_t* arena;
    size_t arena_bytes;
    int G;
    int smem_bytes;
    int t_host;
    std::vector<ushort2> cols;       // [U][depth][4]
    std::vector<uint32_t> goff;      // [G][depth][4] per-GEMM stream offsets (16-B units)
    int lg_on, lg_np;                // logits GEMM planned, and its passes (EngineDev)
    uint32_t* d_goff;
    ushort2* d_cols;
    // arena sub-allocations for per-layer small params
    std::vector<float*> bias_ptr[4];
    std::vector<float*> ln_ptr[4];
    std::vector<__half*> enc_w;      // [2S][W] fp16, transposed copy of c_enc_kv.w
    std::vector<float*> enc_b;
    __half* enc_x16;                 // [max_batch*enc_dims][W] fp16 scratch
    __half* enc_y16;                 // [max_batch*enc_dims][2S] fp16 scratch
    // chunked prefill (prefill.cu): K-major fp16 copies of the four Conv1D weights of every layer and the
    // [pf_rows x .] activation workspace; pf_rows = 0 when the configuration cannot use the tensor-core path
    std::vector<__half*> wt[4];      // [N][K]
    int pf_rows, pf_len;             // workspace rows (= max_batch * pf_len), positions per prefill
    __half *pf_x, *pf_xn, *pf_qkv, *pf_a, *pf_x1, *pf_g;
};
