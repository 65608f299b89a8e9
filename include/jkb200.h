/*
 * jkb200.h - C ABI of libjkb200.so: H100 (sm_90a) kernels for Jukebox's sampling hot path.
 *
 * Boundary contract (SURVEY.md section 8b):
 *   - plain C: pointers, sizes, cudaStream_t (passed as void*); no torch types
 *   - every call enqueues on the given stream and returns; nothing synchronises, nothing
 *     allocates or frees caller memory.  Engines live inside a caller-provided arena whose
 *     size is reported by the *_arena_bytes call.
 *   - return value 0 = ok, negative = error; jk_last_error() gives the message
 *     (thread-local).  The Python host turns a non-zero code into RuntimeError, the same
 *     way the reference's optional native plug-ins surface C++ exceptions
 *     (apex/csrc/layer_norm_cuda.cpp:138-159 -> RuntimeError in jukebox/transformer/ops.py:8-24).
 *
 * Each entry point cites the reference interface it replaces (paths under /root/reference/jukebox).
 */
#ifndef JKB200_H
#define JKB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define JK_MAX_DEPTH 96
#define JK_MAX_BATCH 32

typedef void* jk_stream_t;          /* cudaStream_t */

const char* jk_last_error(void);
int jk_version(void);
/* number of SMs of the current device (grid size of the persistent decode kernel) */
int jk_device_sm_count(int* out);

/* ------------------------------------------------------------------------------------------
 * Autoregressive prior decode engine.
 *
 * Replaces the per-token body of ConditionalAutoregressive2D.sample / primed_sample
 * (prior/autoregressive.py:199-359): get_emb (:177-197) -> Transformer.forward(sample=True)
 * (transformer/transformer.py:169-192) -> ResAttnBlock sample branch (:62-65,82-86) ->
 * LayerNorm (transformer/ops.py:14-24), Conv1D (ops.py:83-101), FactoredAttention.forward with
 * its KV cache (transformer/factored_attention.py:230-301, 328-373), MLP + quick_gelu
 * (transformer.py:19-30, ops.py:33-35) -> +cond -> x_out logits (autoregressive.py:226-229).
 *
 * One jk_prior_step call = one token position for up to 32 samples, executed by ONE persistent
 * kernel (grid = #SMs) that streams every layer's fp16 weights once through a TMA bulk-copy
 * ring in shared memory.  The position is read from device memory, so the call sequence is
 * CUDA-graph capturable.
 * ---------------------------------------------------------------------------------------- */
typedef struct jk_prior_config {
    int32_t width;            /* prior_width                                   */
    int32_t depth;            /* prior_depth                                   */
    int32_t heads;
    int32_t n_state;          /* int(m_attn * width)  (transformer.py:42)      */
    int32_t mlp_width;        /* int(m_mlp * width)                            */
    int32_t n_ctx;            /* full input_dims of the CA2D (incl. lyric tokens for single_enc_dec) */
    int32_t blocks;           /* 0 if none (dense only)                        */
    int32_t bins;             /* rows of x_out; 0 when only_encode             */
    int32_t prime_len;        /* raw prime_len for attn_func 7, else 0         */
    int32_t encoder_dims;     /* rows of the encoder K/V for attn_func 6       */
    int32_t max_batch;        /* <= JK_MAX_BATCH                                */
    int32_t add_cond_after;   /* 1 unless merged_decoder (autoregressive.py:87-93) */
    int32_t attn_func[JK_MAX_DEPTH];  /* per layer: 0,1,2,3,6,7 (transformer.py:110-124) */
} jk_prior_config;

/* Reference-layout weights of one ResAttnBlock, device pointers.  *_w are Conv1D.w
 * [n_in, n_out] row-major (ops.py:89-95) in fp32 (w_dtype 0) or fp16 (w_dtype 1, fp16_params);
 * biases and LayerNorm parameters are fp32 (biases may be fp16 when b_dtype is 1). */
typedef struct jk_layer_weights {
    const void* c_attn_w;  const void* c_attn_b;      /* [W, 3S] ([W, S] for attn_func 6)  */
    const void* c_enc_kv_w; const void* c_enc_kv_b;   /* [W, 2S], attn_func 6 only, else NULL */
    const void* c_proj_w;  const void* c_proj_b;      /* [S, W]                              */
    const void* fc_w;      const void* fc_b;          /* [W, M]                              */
    const void* proj2_w;   const void* proj2_b;       /* [M, W]                              */
    const float* ln0_g; const float* ln0_b;           /* [W]                                 */
    const float* ln1_g; const float* ln1_b;           /* [W]                                 */
    int32_t w_dtype;       /* 0 = fp32, 1 = fp16 */
    int32_t b_dtype;       /* 0 = fp32, 1 = fp16 */
} jk_layer_weights;

typedef struct jk_prior jk_prior;   /* opaque; lives in the caller's arena */

/* How the engine would lay a configuration out on a device with `n_sms` SMs - pure host arithmetic, no device needed
 * (the CPU tests use it; the engine itself always plans for the current device).  cols (optional, uint16 pairs
 * [units][depth][4][2]) receives (first 8-column group, number of groups) of every unit for the four Conv1Ds of a layer,
 * followed by the same pairs of the logits GEMM, [logits_passes][units][2]. */
typedef struct jk_prior_plan_info {
    int32_t k_split;          /* CTAs per unit: they share the unit's columns and split K                 */
    int32_t units;            /* n_sms / k_split                                                          */
    int32_t ring_slots;       /* 16 KB weight-ring slots per SM                                           */
    int32_t smem_bytes;       /* dynamic shared memory of the decode kernel                               */
    int32_t tile_rows;        /* K/V rows per attention tile                                              */
    int32_t logits_passes;    /* passes of the tensor-core logits GEMM (0: fp32 FMA logits)               */
    uint64_t arena_bytes;
    uint64_t stream_stride;   /* bytes of the longest per-SM weight stream (+ padding)                    */
} jk_prior_plan_info;
int jk_prior_plan(const jk_prior_config* cfg, int n_sms, jk_prior_plan_info* out, uint16_t* cols, size_t cols_len);

/* bytes of device memory the engine needs for packed weights, KV caches and activations */
int jk_prior_arena_bytes(const jk_prior_config* cfg, size_t* bytes);
/* `arena` is device memory (256-B aligned) of at least jk_prior_arena_bytes; it is zeroed here */
int jk_prior_create(const jk_prior_config* cfg, void* arena, size_t arena_bytes,
                    jk_prior** out, jk_stream_t stream);
int jk_prior_destroy(jk_prior* p);
/* pack one layer's weights into the per-SM stream layout (device -> device) */
int jk_prior_load_layer(jk_prior* p, int layer, const jk_layer_weights* w, jk_stream_t stream);
/* embeddings are used in place (fp32, reference layout): x_emb [bins_in, W], pos_emb [n_ctx, W],
 * x_out [bins, W] (= x_emb when tied), start_token [W] or NULL */
int jk_prior_set_embeddings(jk_prior* p, const float* x_emb, const float* pos_emb,
                            const float* x_out, const float* start_token);
/* position <- t0 (usually 0); KV caches are logically emptied (FactoredAttention.del_cache,
 * factored_attention.py:375-381) */
int jk_prior_reset(jk_prior* p, int t0, jk_stream_t stream);
/* encoder K/V for attn_func 6 layers: c_enc_kv(encoder_kv) computed once per window
 * (factored_attention.py:273-287).  encoder_kv: fp32 [n, encoder_dims, W] */
/* 1 if this engine multiplies the logits on the tensor cores (hi / lo fp16 split of x_out; needs an even K split and
 * bins > 0), i.e. if jk_step_args.logit_bias is worth computing */
int jk_prior_has_logits_gemm(const jk_prior* p, int* on);

int jk_prior_set_encoder_kv(jk_prior* p, const float* encoder_kv, int n_samples, jk_stream_t stream);

typedef struct jk_step_args {
    int32_t n_samples;            /* <= max_batch */
    /* input: either an embedded activation (Transformer.forward boundary) ... */
    const float* x_in;            /* fp32 [n, W] or NULL */
    /* ... or tokens (CA2D.sample boundary): token fed at position t is tokens[b*tok_stride + t-1] */
    const int64_t* tokens;        /* int64, or NULL */
    int64_t tok_stride;
    const float* y_cond;          /* fp32 [n, W]: input at t == 0 when the prior is y-conditioned, else NULL -> start_token */
    const float* x_cond;          /* fp32 [n, x_cond_len, W] or NULL (treated as zeros) */
    int64_t x_cond_len;           /* 1 or n_ctx */
    /* outputs (any may be NULL) */
    float* h_out;                 /* fp32 [n, W]: Transformer.forward output (before +cond) */
    float* logits;                /* fp32: logits[b*logits_bstride + t*logits_tstride + v] */
    int64_t logits_bstride;
    int64_t logits_tstride;       /* 0 to overwrite the same [n, bins] buffer every step */
    /* optional: x_cond . x_out^T of every position, computed once per window by the caller (the logits are linear in the
     * activation: (h + x_cond) . x_out^T = h . x_out^T + logit_bias).  With it, priors that add x_cond behind the stack
     * (autoregressive.py:226-227: every label-conditioned prior) still take the tensor-core logits product, whose
     * activation operand must be an fp16 value; NULL keeps the fp32 product of h + x_cond.
     * logit_bias[b*logit_bias_bstride + t*logit_bias_tstride + v]; ignored when the engine has no logits GEMM
     * (jk_prior_has_logits_gemm). */
    const float* logit_bias;
    int64_t logit_bias_bstride;
    int64_t logit_bias_tstride;
} jk_step_args;

/* Attention weights of one layer recorded by a prefill call (record_attn in fp16 mode, factored_attention.py:83-105, the
 * pass lyric alignment reads, align.py:91-96).  w: device fp16 [n_samples][heads][n_positions][ld]; w[b][h][q][k] =
 * fp16(softmax_fp32(fp16(fp16(q.k) * dh^-1/2))[k]) for key position k of the layer's pattern (for an encoder-decoder layer
 * k is the encoder row), 0 for every other k; a query without keys (previous-block attention in the first block) is a
 * row of zeros.  Keys >= ld are not written, so a prime layer can keep just its lyric columns (ld = prime_len). */
typedef struct jk_attn_record {
    int32_t layer;
    int32_t ld;
    void* w;
} jk_attn_record;

/* Activations of one layer returned by a prefill call (the representations of JukeMIR: a prior's intermediate layer,
 * averaged over time).  After layer `layer`'s MLP residual add, the fp16 residual stream of positions [t0, t1) of every
 * sample is taken in fp32, plus the call's own x_cond (x_cond_len 1 or n_ctx) when add_x_cond is set:
 *   pool = 0: out fp32 [n_samples, t1 - t0, width];
 *   pool = 1: out fp32 [n_samples, width], the mean over those positions.
 * The mean sums in fp64 in an order that depends on neither the batch nor the device, so a sample's row has the same
 * bits alone and in any batch; jk_pool_rows_f32 is the same kernel over fp32 rows.  out must be 16-byte aligned.  A layer
 * out of range (or >= n_layers when truncating), listed twice, an empty or out-of-range [t0, t1), a NULL out or
 * add_x_cond without x_cond is an error, and nothing is written. */
typedef struct jk_act_capture {
    int32_t layer;
    int32_t t0, t1;
    int32_t pool;
    int32_t add_x_cond;
    float* out;
} jk_act_capture;

/* Chunked prefill of the given (prime) tokens: positions 0 .. n_positions-1 of every sample through all
 * layers in one call - the chunked half of ConditionalAutoregressive2D.primed_sample
 * (prior/autoregressive.py:251-359), whose own check_chunks asserts it equals stepping token by token.
 * The four Conv1Ds of each layer run as [n_samples * n_positions, K] x [K, N] GEMMs on wgmma.  On return
 * the engine stands at position n_positions (K/V caches filled), exactly as after that many jk_prior_step
 * calls.  tokens[b * tok_stride + t] is the token AT position t (the input of position t+1), as in
 * jk_step_args; h_out (optional, fp32 [n_samples, n_positions, width]) receives the transformer output -
 * the `only_encode` forward of the lyric encoder (prior/prior.py:285-301).
 * Continuation: an engine at position t0 > 0 (after steps, a prefill or a jk_prior_select) runs positions
 * t0 .. t0+n_positions-1 of its first n_samples rows on top of their K/V caches and then stands at t0 + n_positions,
 * as after that many more jk_prior_step calls.  Row i of h_out is then position t0 + i; the embedding of position t
 * reads tokens[b * tok_stride + t - 1], pos_emb and x_cond (x_cond_len n_ctx) at t, and y_cond is not read (it feeds
 * position 0 only).  t0 + n_positions > n_ctx, n_positions beyond the capacity, an engine whose last prefill stopped
 * early, and record, capture or a truncating n_layers with t0 > 0 are errors: nothing is launched and the position
 * stays. */
typedef struct jk_prefill_args {
    int32_t n_samples;
    int32_t n_positions;
    const int64_t* tokens;
    int64_t tok_stride;
    const float* y_cond;      /* [n_samples, width] or NULL (start token) */
    const float* x_cond;      /* [n_samples, x_cond_len, width] or NULL */
    int64_t x_cond_len;       /* 1 or n_ctx */
    float* h_out;
    const jk_attn_record* record;   /* n_record distinct layers whose weights this call records, or NULL */
    int32_t n_record;
    /* 0: every layer.  1 <= n_layers < depth: layers 0 .. n_layers-1 only (h_out is then the last of them).  Such a
     * truncated call leaves the later layers' K/V caches unfilled, so the engine cannot go on: jk_prior_position
     * reports -1 and jk_prior_step / jk_prior_prefill return an error until jk_prior_reset.  n_layers == depth is a
     * full call. */
    int32_t n_layers;
    const jk_act_capture* capture;           /* n_capture distinct layers whose activations this call returns, or NULL */
    int32_t n_capture;
} jk_prefill_args;

/* out[b, :] = mean over t in [t0, t1) of (x[b, t, :] (+ x_cond[b, x_cond_len > 1 ? t : 0, :])), x fp32 [n, P, width],
 * x_cond fp32 [n, x_cond_len, width] or NULL (x_cond_len 1 or >= t1), out fp32 [n, width], 16-byte aligned: the pooling
 * of jk_act_capture for rows computed elsewhere (the fp32 path), the same kernel and summation order. */
int jk_pool_rows_f32(const float* x, int n, int P, int width, int t0, int t1, const float* x_cond, int64_t x_cond_len,
                     float* out, jk_stream_t stream);
/* positions one prefill call can take; 0 when the configuration has no tensor-core prefill (a GEMM K that
 * is not a multiple of 64, or encoder-decoder layers): step the given tokens instead */
int jk_prior_prefill_capacity(const jk_prior* p, int* max_positions);
/* the same number for an engine of this configuration on the current device, from host arithmetic alone (no engine is
 * built): callers that choose between the prefill and another path ask before building one.  An error when the
 * configuration cannot make an engine (jk_prior_arena_bytes would fail). */
int jk_prior_config_prefill_capacity(const jk_prior_config* cfg, int* max_positions);
int jk_prior_prefill(jk_prior* p, const jk_prefill_args* args, jk_stream_t stream);

/* The attention of one prefill layer on its own: the code jk_prior_prefill runs per layer (forward output and recorded
 * weights), for tests and for callers that hold q / K / V themselves.  Per sample b, head h and query position p < P,
 * over the keys of p's pattern (attn_func 0 dense, 1 block, 2 transpose, 3 previous block, 7 prime: positions < P;
 * 6 encoder-decoder: every encoder row):
 *   s_j = fp16(fp16(q . k_j) * dh^-1/2);  out = fp16(sum_j fp16(exp(s_j - max s)) v_j / sum_j exp(s_j - max s))
 * (exponentials fp32; a query without keys gives 0) and, when w is set, the weights of jk_attn_record. */
typedef struct jk_prefill_attn_args {
    const void* qkv;          /* fp16 [n * P][q_stride]: q | k | v of each row, q_stride = 3 * heads * dh (attn_func 6:
                                 q only, q_stride = heads * dh) */
    const void* k_cache;      /* attn_func 6: fp16 [n][heads][enc_rows][dh_pad]; else NULL */
    const void* v_cache;
    void* out;                /* fp16 [n * P][heads * dh], or NULL */
    void* w;                  /* recorded weights, fp16 [n][heads][P][ld], or NULL (zeroed first, keys >= ld skipped) */
    int32_t ld;
    int32_t n, P, heads, dh, dh_pad;   /* dh_pad: row length of the caches, dh <= dh_pad, a multiple of 16 */
    int32_t attn_func, bc, prime;      /* bc: block length (1, 2, 3); prime: the padded prime length (7) */
    int32_t enc_rows;                  /* attn_func 6: encoder rows of the caches */
    int32_t route;                     /* 0: the prefill's own choice of kernel; 1: the scalar kernels */
    /* Continuation (q_offset > 0 or cache_rows > 0), as jk_prior_prefill runs an engine at position q_offset: query row
     * i is position q_offset + i, and the keys (and values) of every pattern are read from k_cache / v_cache,
     * fp16 [n][heads][cache_rows][dh_pad] in the decode engine's layout (DESIGN §4): position p's keys are cache rows
     * base(p) + j, j < the pattern's key count at p, with base 0 (0, 1, 7), (p % bc) * blocks (2) or
     * ((p / bc + 1) % 2) * bc (3).  qkv then holds q only in its first third (K / V columns are not read).  w must be
     * NULL; cache_rows must cover the rows the pattern reads, and attn_func 2 needs blocks >= 1 with
     * q_offset + P <= bc * blocks.  Both 0: the head of a window, as above. */
    int32_t q_offset;
    int32_t cache_rows;
    int32_t blocks;
} jk_prefill_attn_args;
/* the kernels a call ran: tensor_cores 0 = the scalar kernels (tile_dh, stage_bytes 0); 1 = mma.sync kernels of head
 * tile tile_dh (32, 64, 128, 160, 256) staging K / V in stage_bytes (16 or 4) chunks */
typedef struct jk_prefill_attn_route {
    int32_t tensor_cores;
    int32_t tile_dh;
    int32_t stage_bytes;
} jk_prefill_attn_route;
/* qkv, out and the caches must be 16-byte aligned; neither out nor w, an unknown attn_func, a pattern parameter < 1,
 * dh > dh_pad or dh_pad % 16 != 0, or a scalar-route shape with (dh + max(q_offset + P, enc_rows)) * 4 > 64 KB is an
 * error, and nothing is written.  taken (may be NULL) receives the route. */
int jk_prefill_attention_f16(const jk_prefill_attn_args* a, jk_prefill_attn_route* taken, jk_stream_t stream);

/* one token position; increments the device-side position counter */
int jk_prior_step(jk_prior* p, const jk_step_args* a, jk_stream_t stream);

/* Sample selection (csrc/select.cu): row b of the engine becomes a copy of row parents[b], b < n, so that one sample's
 * history can be continued in several rows (a prime prefilled once and repeated, or the likeliest samples of a window
 * kept).  The state a row carries from one step to the next is its K / V cache in every layer, the encoder-decoder (6)
 * and prime (7) layers included; everything else an engine holds is rebuilt by every step.
 * jk_prior_select_plan is host arithmetic (no device needed): the rows to stash (read by another row AND overwritten,
 * ascending) and the workspace they need.  Broadcasting one row, or keeping some rows in place and copying them to the
 * others, stashes nothing; only a permutation that overwrites a row another row still reads does.  n in [1, max_batch]
 * and every parent in [0, n), else an error. */
typedef struct jk_select_plan_info {
    int32_t n_copies;                 /* rows b with parents[b] != b                                    */
    int32_t n_stash;                  /* rows copied to the workspace first                             */
    int32_t stash[JK_MAX_BATCH];      /* those rows, ascending; slot i of the workspace holds stash[i]  */
    uint64_t row_bytes;               /* one row's K and V over every layer                             */
    uint64_t workspace_bytes;         /* n_stash * row_bytes                                            */
    uint64_t bytes_moved;             /* read + written: 2 * row_bytes * (n_stash + n_copies)           */
} jk_select_plan_info;
int jk_prior_select_plan(const jk_prior_config* cfg, const int32_t* parents, int n, jk_select_plan_info* out);
/* Reorders rows [0, n) of every layer's K / V cache in place: at most two launches on `stream` (the stashed rows into
 * `workspace`, then every copy), nothing synchronises.  parents is host memory.  workspace: device memory of at least
 * the plan's workspace_bytes, 16-byte aligned (NULL when that is 0).  A bad n or parent, a short workspace or an engine
 * whose last prefill stopped early (jk_prior_position -1) is an error, and nothing is launched.  The position does not
 * change: every row continues from it. */
int jk_prior_select(jk_prior* p, const int32_t* parents, int n, void* workspace, size_t workspace_bytes,
                    jk_stream_t stream);
/* current position (host copy of the device counter as tracked by the calls made so far); -1 after a truncated prefill
 * (jk_prefill_args.n_layers), until jk_prior_reset */
int jk_prior_position(const jk_prior* p, int* t);
/* profiling buffers of the decode kernel (device ptr and size in halfs; any other `which` is an error):
 * which: 5 = globaltimer stamps (uint64 per phase), 6 = clock64 stamps (int64 [phase][8]), 7 = globaltimer entry / exit
 * stamps of every CTA in the five phases of layer 1 (uint64 [5][256][2]).  Written only when the engine was created with JK_PROFILE set.
 * The activations travel between SMs as flagged words and are not kept: h_out and logits of jk_step_args are the
 * step's observable outputs. */
int jk_prior_debug_buffer(const jk_prior* p, int which, const void** ptr, size_t* n_halfs);

/* Conv1D at prefill / training shape on the tensor cores (wgmma + TMA): y[M, N] = x[M, K] . w + b, fp16 in,
 * fp32 accumulate, fp16 out (transformer/ops.py:83-101).  w_t is the weight TRANSPOSED: [N, K] row-major fp16;
 * bias fp32 [N] or NULL; K >= 64 and K % 8 == 0 (a K tail past the last 64-wide block reads zeros); x, w_t and y
 * 16-byte aligned.  Used for c_enc_kv(encoder_kv) (factored_attention.py:273-287) inside jk_prior_set_encoder_kv. */
int jk_conv1d_prefill_f16(const void* x, const void* w_t, const float* bias, void* y, int M, int N, int K,
                          jk_stream_t stream);
/* The GEMM of the chunked prefill with its epilogues, the same kernel as above; with y = fp16(acc + bias) rounded once:
 *   epi 0: y;   1: quick_gelu with the reference's fp16 roundings (ops.py:33-35),
 *               z = fp16(1.702 y), sg = fp16(1 / (1 + exp(-z))), out = fp16(y * sg);   2: fp16(res + y)
 * res: fp16 [M, N], read by epi 2 only.  K as above; x, w_t, y and res (when set) 16-byte aligned; epi 2 without res,
 * another epi or a constraint not met is an error, checked before anything is launched. */
int jk_prefill_gemm_f16(const void* x, const void* w_t, const float* bias, const void* res, void* y, int M, int N, int K,
                        int epi, jk_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * VQ-VAE.  Tensors are channels-last: [N, T, C] fp32.
 * ---------------------------------------------------------------------------------------- */
/* BottleneckBlock.quantise (vqvae/bottleneck.py:112-119): idx = argmin_j |x|^2 - 2 x.k_j + |k_j|^2
 * in fp32, lowest index on ties.  x [n, width], codebook [k_bins, width], idx int64 [n]. */
int jk_vq_argmin(const float* x, const float* codebook, int64_t* idx, float* min_dist /*nullable*/,
                 int64_t n, int k_bins, int width, jk_stream_t stream);
/* BottleneckBlock.dequantise (bottleneck.py:121-123): out[n, :] = codebook[idx[n], :] */
int jk_vq_gather(const int64_t* idx, const float* codebook, float* out, int64_t n, int k_bins,
                 int width, jk_stream_t stream);

/* Generic channels-last 1-D convolution used for every conv of Encoder/Decoder/Resnet1D
 * (vqvae/encdec.py:6-131, vqvae/resnet.py:27-44) and the upsampler Conditioner
 * (prior/conditioners.py:8-48):
 *   out[n, t, co] = (res ? res[n, t, co] : 0)
 *                 + scale * ( bias[co] + sum_tap sum_ci w[tap, ci, co] * pre(in[n, t*in_stride + tap_off[tap], ci]) )
 * pre = ReLU when relu_in.  Out-of-range input positions read as zero (conv padding).
 * w is packed [n_taps, c_in, c_out] (see jk_pack_conv_weight).  For a transposed conv the caller
 * issues one call per output phase with out_stride 2 / out_offset r. */
typedef struct jk_conv_args {
    const float* in;  int64_t t_in;  int32_t c_in;
    float* out;       int64_t t_out; int32_t c_out;     /* t_out counts positions written by THIS call */
    const float* w;   const float* bias;
    const float* res;                 /* nullable; indexed like out */
    int32_t n_taps;   int32_t tap_off[4];
    int32_t in_stride;                /* input positions per output position (1, or 2 for the strided encoder conv) */
    int32_t out_stride; int32_t out_offset;  /* output row = t*out_stride + out_offset (within a buffer of t_out*out_stride rows) */
    int32_t relu_in;
    float scale;
    int32_t n;                        /* batch */
    int32_t tensor_cores;             /* 0: exact fp32 FMAs in a fixed order (the encoder: its output feeds the bit-exact argmin);
                                         1: decoder side - c_in, c_out in {32, 64} run with the fp16 x 3 split (fp32-level
                                         accuracy, free summation order): on wgmma + TMA for stride-1 inputs of >= 128
                                         positions and <= 3 taps, on mma.sync otherwise; other shapes ignore the flag */
} jk_conv_args;
int jk_conv1d_cl(const jk_conv_args* a, jk_stream_t stream);

/* Wide decoder-side convolutions on the tensor cores (wgmma + TMA): the convs of the upsampler Conditioner
 * (prior/conditioners.py:8-48), c_in and c_out multiples of 64 with one of them above 64.  Same arithmetic contract as
 * tensor_cores = 1 above: every product is the fp16 x 3 split hi.w_hi + lo.w_hi + hi.w_lo with the weights scaled by 2^8
 * before the split, fp32 accumulation, free summation order.
 * jk_pack_conv_weight_split turns a packed fp32 weight [k, c_in, c_out] (jk_pack_conv_weight, or one phase of a
 * transposed conv) into the layout the kernel streams: [hi | lo][c_out][k * c_in] fp16, jk_conv_weight_split_bytes bytes
 * of device memory (16-byte aligned).  Do it once per weight load.
 * jk_conv1d_tc_wide computes what jk_conv1d_cl documents, reading the weight from w_split; a->w and a->tensor_cores are
 * not read (the exact route is jk_conv1d_cl with tensor_cores = 0 and the packed weight).  It takes in_stride 1,
 * 1..3 taps, t_in >= 128 and 16-byte aligned in / out / bias / res, and returns an error naming the constraint otherwise:
 * callers keep jk_conv1d_cl for those shapes. */
int jk_conv_weight_split_bytes(int k, int c_in, int c_out, size_t* bytes);
int jk_pack_conv_weight_split(const float* packed, void* split, int k, int c_in, int c_out, jk_stream_t stream);
int jk_conv1d_tc_wide(const jk_conv_args* a, const void* w_split, jk_stream_t stream);

/* ResConv1DBlock (vqvae/resnet.py:27-44): out = x + res_scale * (W2.relu(W1 *_dil relu(x) + b1) + b2)
 * x, out [n, T, C] (x != out); w1 packed [3, C, Cs]; w2 packed [1, Cs, C].  For C == Cs in {32, 64} (every
 * ResConv1DBlock of the reference's VQ-VAEs) with x, out, w1, w2, b1 and b2 16-byte aligned this is ONE launch with the
 * hidden activation kept in shared memory and tmp may be NULL; other shapes and pointers run as two jk_conv1d_cl launches
 * through tmp [n, T, Cs], and without tmp they are an error. */
int jk_resblock_cl(const float* x, float* out, float* tmp, const float* w1, const float* b1, const float* w2,
                   const float* b2, int n, int64_t T, int C, int Cs, int dilation, float res_scale,
                   jk_stream_t stream);

/* The same ResConv1DBlock on the tensor cores for the DECODER side (Decoder stacks of vqvae/encdec.py:87-131 and the
 * upsampler Conditioner, prior/conditioners.py:8-48), C == Cs in {32, 64}: fp16 x 3 split (hi / lo fp16 operands, weights
 * scaled by 2^8 before their split, hi.w_hi + lo.w_hi + hi.w_lo accumulated in fp32), on wgmma + TMA for T >= 128, on
 * mma.sync m16n8k16 for shorter clips; i.e. fp32 accuracy up to the dropped lo.w_lo term but NOT the FMA order of
 * jk_resblock_cl.  x and out must be 16-byte aligned and b1, b2 8-byte aligned; other pointers are an error (nothing is
 * launched).  The encoder, whose output feeds the bit-exact codebook argmin, must keep jk_resblock_cl. */
int jk_resblock_tc(const float* x, float* out, const float* w1, const float* b1, const float* w2, const float* b2,
                   int n, int64_t T, int C, int dilation, float res_scale, jk_stream_t stream);

/* Spectral losses of VQVAE.forward (utils/audio_utils.py:80-131), one fused kernel: no spectrogram reaches memory.
 * Per clip n of two mono signals a, b [n, T] fp32 (torch.stft semantics of audio_utils.py:80-84: center=True with
 * reflect padding of n_fft/2, `window` = the periodic Hann of win_length centred in n_fft at (n_fft - win_length)/2,
 * onesided, 1 + T/hop frames):
 *   resid[n]  = sum over frames and bins of (|STFT(a_n)| - |STFT(b_n)|)^2
 *   norm_a[n] = sum over frames and bins of  |STFT(a_n)|^2            (both float64)
 * n_fft a power of two in [256, 4096], 1 <= win_length <= n_fft, hop >= 1, T > n_fft/2; anything else is an error.
 * workspace: device memory of jk_stft_workspace_bytes(n, T, n_fft, hop) bytes (8-byte aligned; 0 for invalid sizes).
 * The result is bitwise deterministic and the same for a clip whatever the batch it is computed in. */
int     jk_stft_mag_diff(const float* a, const float* b, const float* window, double* resid, double* norm_a,
                         int n, int64_t T, int n_fft, int hop, int win_length,
                         void* workspace, size_t workspace_bytes, jk_stream_t stream);
size_t  jk_stft_workspace_bytes(int n, int64_t T, int n_fft, int hop);

/* Token sampling of the autoregressive loop (prior/autoregressive.py:233-235, 343-345):
 *   tokens[r, position] ~ Categorical(logits = logits[r, :] / temp),  r = 0..n-1
 * one launch per position.  logits: fp32 rows `logits_stride` floats apart (entries of -inf carry no
 * mass, so rows already passed through filter_logits are valid input); tokens: int64 [n, tok_stride].
 * The uniform behind row r at `position` is Philox4x32-10(key = seed, counter = (position, r)), so a
 * (seed, position, row) triple always draws the same token for the same logits. */
int jk_sample_categorical(const float* logits, int64_t logits_stride, int n, int bins, float temp,
                          uint64_t seed, int position, int64_t* tokens, int64_t tok_stride,
                          jk_stream_t stream);
/* The same draw, scored in the same launch.  logits: what jk_sample_categorical would take (the engine's row, or the
 * filter_logits output with temp 1); the token drawn is bit-identical to jk_sample_categorical's for the same
 * arguments.  logits == NULL: nothing is drawn, tokens[r, position] is given.  Either way
 *   logp[r * logp_stride + position] = log_softmax(raw[r, :])[token]     (fp32)
 * the log-likelihood at temperature 1 of the raw, unfiltered logits (raw: fp32 rows raw_stride floats apart); nan for a
 * given token outside [0, bins). */
int jk_sample_categorical_scored(const float* logits, int64_t logits_stride, const float* raw, int64_t raw_stride,
                                 int n, int bins, float temp, uint64_t seed, int position, int64_t* tokens,
                                 int64_t tok_stride, float* logp, int64_t logp_stride, jk_stream_t stream);

/* Log-probabilities of given tokens from the activations, with no logits tensor (csrc/score.cu):
 *   logp[m] = z[m, targets[m]] - lse[m],  lse[m] = log sum_b exp(z[m, b]),  z = h . x_out^T
 * h: fp32 [m, width] (x_cond already added when the prior adds it behind the stack), width a multiple of 64; targets:
 * int64 [m]; logp, and lse unless NULL: fp32 [m].  The product is the fp16 x 3 split (hi.w_hi + hi.w_lo + lo.w_hi,
 * fp32 accumulation promoted every 64 channels) on the tensor cores, x_out scaled by 2^8 before its split.
 * jk_pack_xout_split turns x_out fp32 [bins, width] (nn.Linear layout) into the layout the kernel streams,
 * jk_xout_split_bytes bytes of 16-byte aligned device memory; do it once per weight load.  It returns an error when a
 * weight lies outside what the scaled split holds (|w| > 255.9, inf, nan).
 * jk_xout_logprob needs jk_xout_logprob_workspace_bytes of 256-byte aligned device memory and a 16-byte aligned h.  It
 * synchronises the stream to report its range check: an activation with |h| > 65504 or not finite, or a target outside
 * [0, bins), is an error (the outputs of the call are then nan, never a wrong number).  A row's result does not depend
 * on the other rows: it is bitwise the same alone and in any batch. */
int jk_xout_split_bytes(int bins, int width, size_t* bytes);
int jk_pack_xout_split(const float* w, void* split, int bins, int width, jk_stream_t stream);
int jk_xout_logprob_workspace_bytes(int m, int width, int bins, size_t* bytes);
int jk_xout_logprob(const float* h, int m, int width, const void* w_split, int bins, const int64_t* targets,
                    float* logp, float* lse, void* workspace, size_t workspace_bytes, jk_stream_t stream);

/* Statistics of the predictive distribution p = softmax(z) from the activations, with no logits tensor (csrc/score.cu):
 *   entropy[m]           = lse[m] - sum_b p[m, b] z[m, b]                      (nats; fp32, accumulated in fp64)
 *   logp[m]              = z[m, targets[m]] - lse[m]                           (when targets is given)
 *   topk_ids[m, 0..k)    = the k bins of largest z[m, :], by descending z, ties to the lower bin   (int64)
 *   topk_logp[m, 0..k)   = z[m, topk_ids[m, j]] - lse[m]
 *   lse[m]               = log sum_b exp(z[m, b])
 * h, width, w_split (jk_pack_xout_split's layout) and the product are jk_xout_logprob's; logp and lse are its results bit
 * for bit.  targets and logp are both NULL or both given; topk_ids and topk_logp may each be NULL (k = 0: no top-k);
 * lse may be NULL; 0 <= k <= JK_XOUT_STATS_MAX_K and k <= bins.  It needs jk_xout_stats_workspace_bytes of 256-byte
 * aligned device memory and synchronises the stream for the same range check as jk_xout_logprob: an out-of-range
 * activation or target is an error, and the outputs are then nan (ids -1), never a wrong number.  A row's result does not
 * depend on the other rows. */
#define JK_XOUT_STATS_MAX_K 16
int jk_xout_stats_workspace_bytes(int m, int width, int bins, int k, size_t* bytes);
int jk_xout_stats(const float* h, int m, int width, const void* w_split, int bins, const int64_t* targets, int k,
                  float* logp, float* entropy, int64_t* topk_ids, float* topk_logp, float* lse, void* workspace,
                  size_t workspace_bytes, jk_stream_t stream);

/* top-k / nucleus filtering in front of the sampler (transformer/ops.py:113-142 `filter_logits`, applied to
 * logits / temp as autoregressive.py:232-234 does): out[r, v] = logits[r, v] / temp if v stays, else -inf.
 * top_k > 0: the k largest stay; top_p > 0: the smallest prefix of the sorted row whose softmax mass exceeds top_p
 * stays (the entry that crosses the threshold included).  Exactly one of the two must be set; bins <= 4096.
 * Ties at the cut stay together (the reference's scatter-by-index keeps an arbitrary subset of equal values). */
int jk_filter_logits(const float* logits, int64_t logits_stride, int n, int bins, float temp, int top_k,
                     float top_p, float* out, int64_t out_stride, jk_stream_t stream);

/* Guided draw from two conditionings (classifier-free guidance, or a blend of two conditionings), one launch per position.
 * For pair r = 0..n-1, with c[r] the conditional logits (rows c_stride floats apart) and u[r] the alternative ones (rows
 * u_stride apart):
 *   g = c[r] + s (c[r] - u[r])          fp32, each operation rounded to nearest on its own (no FMA): torch's
 *                                       `c + s * (c - u)` gives the same bits
 *   tokens[r, position] = tokens_alt[r, position] ~ Categorical(filter(g / temp))
 * filter: top_k / top_p as jk_filter_logits (at most one set; neither: no filter), and the draw is jk_sample_categorical's
 * (Philox counter (position, r)), so the token equals jk_filter_logits + jk_sample_categorical of g bit for bit.  s = 0
 * gives g = c.  raw and logp are both NULL or both given: logp[r * logp_stride + position] = log_softmax(raw[r])[token],
 * raw rows c_stride floats apart (raw == c: the conditional model's own likelihood at temperature 1, read with c).
 * tokens / tokens_alt: int64 rows tok_stride / tok_alt_stride apart.  bins <= 4096, s finite, temp > 0, n >= 0.  Each
 * operand row is read once; pairs are independent. */
int jk_sample_guided(const float* c, int64_t c_stride, const float* u, int64_t u_stride, int n, int bins, float s,
                     float temp, int top_k, float top_p, uint64_t seed, int position, int64_t* tokens, int64_t tok_stride,
                     int64_t* tokens_alt, int64_t tok_alt_stride, const float* raw, float* logp, int64_t logp_stride,
                     jk_stream_t stream);

/* torch Conv1d weight [c_out, c_in, k] (transposed = 0) or ConvTranspose1d weight
 * [c_in, c_out, k] (transposed = 1) -> packed [k, c_in, c_out] */
int jk_pack_conv_weight(const float* w, float* packed, int c_out, int c_in, int k, int transposed,
                        jk_stream_t stream);

/* LayerNorm over the last dim of fp32 rows (Conditioner.ln, prior/conditioners.py:47;
 * transformer/ops.py:14-24): y = (x-mu)/sqrt(var+eps)*g + b */
int jk_layernorm_f32(const float* x, const float* g, const float* b, float* y, int64_t rows, int width,
                     float eps, jk_stream_t stream);
/* out[n, :] = table[idx[n], :] (+ add[n, :] if add) - embedding lookups of Conditioner /
 * LabelConditioner (prior/conditioners.py:40-43, 57-68) */
int jk_embedding_f32(const int64_t* idx, const float* table, const float* add, float* out, int64_t n,
                     int rows, int width, jk_stream_t stream);

/* ---- fp32 transformer path (not the hot path: exactness against the reference's fp32 outputs) ------------------------
 * Transformer.forward in fp32 (transformer/transformer.py:169-192): sample = forward mode over a whole sequence
 * (training-shaped calls, alignment with record_attn - prior/prior.py:327-344) and sampling with fp32 K/V caches
 * (ConditionalAutoregressive2D.sample(fp16=False), prior/autoregressive.py:199-249).  One structure per layer holds the
 * reference's parameter tensors (fp32, Conv1D layout [n_in, n_out], transformer/ops.py:83-101) and the layer's caches. */
typedef struct jk_f32_layer {
    const float *ln0_g, *ln0_b, *ln1_g, *ln1_b;
    const float *c_attn_w, *c_attn_b;       /* [width, 3 n_state]; [width, n_state] (c_attn of an enc-dec layer) */
    const float *c_enc_kv_w, *c_enc_kv_b;   /* [width, 2 n_state], attn_func 6 only */
    const float *c_proj_w, *c_proj_b;       /* [n_state, width] */
    const float *fc_w, *fc_b;               /* [width, mlp_width] */
    const float *proj2_w, *proj2_b;         /* [mlp_width, width] */
    float *k_cache, *v_cache;               /* [n, n_ctx, n_state] ([n, encoder_dims, n_state] for attn_func 6); rows are
                                               absolute positions.  Forward mode passes scratch of the same shape. */
    float *attn_w;                          /* optional: attention weights [n, heads, P, n_ctx | encoder_dims] of this call
                                               (record_attn, factored_attention.py:100-102), or NULL */
    int32_t attn_func;                      /* 0, 1, 2, 3, 6, 7 (factored_attention.py:49-58) */
} jk_f32_layer;

typedef struct jk_f32_args {
    int32_t n, P, p0;              /* samples, positions in this call, absolute position of the first one */
    int32_t width, n_state, mlp_width, heads, n_ctx, blocks, prime_len, encoder_dims, depth;
    float* x;                      /* [n, P, width]: residual stream, transformed in place */
    const float* encoder_kv;       /* [n, encoder_dims, width] or NULL (read when p0 == 0) */
    float* work;                   /* jk_f32_workspace_floats() floats */
} jk_f32_args;

int jk_f32_workspace_floats(const jk_f32_args* a, size_t* floats);
/* Positions [p0, p0 + P) of every sample through all `depth` layers.  K / V of the new positions are written to the
 * caches first, each query then attends the cache rows of its pattern; a call with p0 = 0, P = n_ctx is the reference's
 * forward mode, P = 1 its per-token sampling step. */
int jk_f32_forward(const jk_f32_args* a, const jk_f32_layer* layers, jk_stream_t stream);
/* x[b, i, :] = (position p0+i == 0 ? y_cond[b] or start_token : x_emb[tokens[b, p0+i-1]]) + pos_emb[p0+i] (+ x_cond)
 * (prior/autoregressive.py:115-123 shifted input in forward mode, :176-191 get_emb in sampling). x_cond_len: 0 = none,
 * 1 = one broadcast row per sample, else rows indexed by position. */
int jk_f32_embed(float* x, const int64_t* tokens, int64_t tok_stride, const float* y_cond, const float* x_cond,
                 int64_t x_cond_len, const float* x_emb, const float* pos_emb, const float* start_token, int n, int P,
                 int p0, int width, jk_stream_t stream);
/* y[M, N] = x[M, K] . w + b;  w is [K, N] (Conv1D) or, with w_is_nk, [N, K] (nn.Linear: x_out, autoregressive.py:86) */
int jk_f32_linear(const float* x, const float* w, const float* b, float* y, int M, int N, int K, int w_is_nk,
                  jk_stream_t stream);

/* ---- gradients of the fp32 path (fine-tuning a prior's decoder) --------------------------------------------------------
 * Deterministic kernels: no atomics on any gradient sum, so two identical calls give bit-identical results.  Every
 * gradient is ADDED to what its buffer holds (.grad accumulates over micro-batches and over the tied x_emb / x_out).
 * One structure per layer mirrors jk_f32_layer's parameters; NULL = frozen, its weight-gradient work is skipped. */
typedef struct jk_f32_grad_layer {
    float *ln0_g, *ln0_b, *ln1_g, *ln1_b;
    float *c_attn_w, *c_attn_b;
    float *c_enc_kv_w, *c_enc_kv_b;
    float *c_proj_w, *c_proj_b;
    float *fc_w, *fc_b;
    float *proj2_w, *proj2_b;
} jk_f32_grad_layer;

int jk_f32_backward_workspace_floats(const jk_f32_args* a, size_t* floats);
/* Backward of jk_f32_forward over a whole window (p0 = 0, P = n_ctx) through layers depth-1 .. 0 of the table.  Each
 * layer's forward is recomputed from saved_inputs[l] ([n, P, width], the layer's input), then differentiated.  dx holds
 * dL/d(output of the last layer) on entry and dL/d(input of layer 0) on return.  a->x is not read; a->work holds
 * jk_f32_backward_workspace_floats() floats; a->encoder_kv is read by enc-dec layers.  d_encoder_kv ([n, encoder_dims,
 * width], or NULL) receives the enc-dec layers' gradient of encoder_kv, added.  All arguments are checked first. */
int jk_f32_backward(const jk_f32_args* a, const jk_f32_layer* layers, const jk_f32_grad_layer* grads,
                    const float* const* saved_inputs, float* dx, float* d_encoder_kv, jk_stream_t stream);
/* dw[K, N] (+)= x[M, K]^T . dy[M, N] and db[N] (+)= sum_m dy[m, :] (either may be NULL): a Conv1D's weight gradient.
 * Also nn.Linear's ([N, K] weight) with x and dy swapped. */
int jk_f32_linear_wgrad(const float* x, const float* dy, float* dw, float* db, int M, int K, int N, int accumulate,
                        jk_stream_t stream);
/* Gradients of jk_f32_embed's tables from dh = dL/dx [n, P, width] (p0 = 0, no x_cond): d_x_emb [bins, width] by token
 * id (pairs sorted once, then summed per id in row order; work holds 2 n (P-1) ints), d_pos_emb [P, width] (sum over
 * items), d_start_token [width] (position 0 of every item; NULL when the prior has y_cond).  Any may be NULL. */
int jk_f32_embed_backward(const float* dh, const int64_t* tokens, int64_t tok_stride, int n, int P, int width, int bins,
                          float* d_x_emb, float* d_pos_emb, float* d_start_token, int* work, int accumulate,
                          jk_stream_t stream);
/* Cross-entropy head over logits [M, bins] (jk_f32_linear's x_out product): loss[m] = logsumexp - logits[m, target]
 * (nats), and logits overwritten with row_weight[m] (softmax - onehot(target)), the gradient of sum_m w_m loss_m. */
int jk_f32_xent_backward(float* logits, const int64_t* targets, const float* row_weight, float* loss, int M, int bins,
                         jk_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* JKB200_H */
