// Sample selection on the decode engine (jk_prior_select, include/jkb200.h): rows of every layer's K / V cache become
// copies of other rows, so one history continues in several rows.  DESIGN.md §4.1.
//
// A row's K (or V) in layer l is one contiguous slab of the [Bmax][H][rows][dh_pad] fp16 cache: H * rows * dh_pad * 2
// bytes at row * slab.  A launch copies the slabs of every (layer, K|V) for a list of (source, destination) row pairs,
// where either side may instead be a stash slot of the caller's workspace (one row's slabs, laid end to end).  The
// grid is (chunks of one row, pairs): a CTA copies one chunk of at most kChunk bytes of one slab with 16-byte loads,
// four in flight per thread.
#include "engine.cuh"

#include <cstring>

using namespace jk;

namespace {

constexpr int kSelThreads = 256;
constexpr unsigned kChunk = 64 * 1024;        // bytes per CTA: 16 loads of 16 bytes per thread
constexpr int kMaxSeg = 2 * JK_MAX_DEPTH;     // (layer, K | V) slabs of a row

struct SelectLaunch {
    int n_seg;
    int8_t src[JK_MAX_BATCH], dst[JK_MAX_BATCH];      // >= 0: a cache row;  v < 0: stash slot -1 - v
    unsigned first[kMaxSeg + 1];                      // first chunk of slab s within a row; first[n_seg]: chunks per row
    unsigned long long ws_off[kMaxSeg];               // offset of slab s within a stash slot
    unsigned long long row_bytes;                     // one stash slot
    uint8_t* ws;
};

__global__ void __launch_bounds__(kSelThreads) select_copy_kernel(const EngineDev* __restrict__ E, const SelectLaunch a) {
    const unsigned c = blockIdx.x;
    int lo = 0, hi = a.n_seg - 1;                     // the slab of chunk c: the last s with first[s] <= c
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.first[mid] <= c) lo = mid; else hi = mid - 1;
    }
    const int s = lo;
    const LayerDev& LD = E->layer[s >> 1];
    const size_t slab = (size_t)E->H * LD.rows * E->dh_pad * 2;
    const size_t off = (size_t)(c - a.first[s]) * kChunk;
    const size_t n16 = (slab - off < kChunk ? slab - off : (size_t)kChunk) / 16;
    uint8_t* cache = (uint8_t*)((s & 1) ? LD.vc : LD.kc);
    const int sr = a.src[blockIdx.y], dr = a.dst[blockIdx.y];
    const uint8_t* from = sr >= 0 ? cache + (size_t)sr * slab + off : a.ws + (size_t)(-1 - sr) * a.row_bytes + a.ws_off[s] + off;
    uint8_t* to = dr >= 0 ? cache + (size_t)dr * slab + off : a.ws + (size_t)(-1 - dr) * a.row_bytes + a.ws_off[s] + off;
    const uint4* __restrict__ f4 = (const uint4*)from;
    uint4* __restrict__ t4 = (uint4*)to;
    for (size_t i = threadIdx.x; i < n16; i += 4 * kSelThreads) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (i + u * kSelThreads < n16) v[u] = __ldg(f4 + i + u * kSelThreads);
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (i + u * kSelThreads < n16) t4[i + u * kSelThreads] = v[u];
    }
}

// bytes of one row's K (or V) in each layer; an error for a configuration the engine would refuse in the same way
int row_slabs(const jk_prior_config& c, size_t* slab) {
    JK_REQUIRE(c.depth >= 1 && c.depth <= JK_MAX_DEPTH, "depth %d out of range", c.depth);
    JK_REQUIRE(c.max_batch >= 1 && c.max_batch <= JK_MAX_BATCH, "max_batch %d out of range (<= %d)", c.max_batch, JK_MAX_BATCH);
    JK_REQUIRE(c.heads >= 1 && c.n_state >= c.heads && c.n_state % c.heads == 0, "n_state %d not a multiple of heads %d",
               c.n_state, c.heads);
    JK_REQUIRE(c.blocks >= 0 && (c.blocks == 0 || c.n_ctx % c.blocks == 0), "n_ctx %% blocks != 0");
    const int dh_pad = head_dim_pad(c), bc = block_len(c), prime_pad = prime_pad_len(c);
    for (int l = 0; l < c.depth; ++l) {
        const int rows = cache_rows_for(c, c.attn_func[l], bc, prime_pad);
        JK_REQUIRE(rows >= 0, "layer %d: attn_func %d has no decode path", l, c.attn_func[l]);
        slab[l] = (size_t)c.heads * rows * dh_pad * 2;
    }
    return 0;
}

int plan(const jk_prior_config& c, const int32_t* parents, int n, jk_select_plan_info* out, size_t* slab) {
    JK_REQUIRE(parents && out, "null argument");
    JK_REQUIRE(n >= 1 && n <= c.max_batch, "n %d out of range [1, max_batch %d]", n, c.max_batch);
    for (int b = 0; b < n; ++b)
        JK_REQUIRE(parents[b] >= 0 && parents[b] < n, "parents[%d] = %d outside [0, %d)", b, parents[b], n);
    int rc = row_slabs(c, slab);
    if (rc) return rc;
    memset(out, 0, sizeof(*out));
    bool read[JK_MAX_BATCH] = {};
    for (int b = 0; b < n; ++b)
        if (parents[b] != b) { out->n_copies += 1; read[parents[b]] = true; }
    for (int r = 0; r < n; ++r)
        if (read[r] && parents[r] != r) out->stash[out->n_stash++] = r;
    for (int l = 0; l < c.depth; ++l) out->row_bytes += 2 * (uint64_t)slab[l];
    out->workspace_bytes = out->row_bytes * out->n_stash;
    out->bytes_moved = 2 * out->row_bytes * (uint64_t)(out->n_stash + out->n_copies);
    return 0;
}

}  // namespace

extern "C" int jk_prior_select_plan(const jk_prior_config* cfg, const int32_t* parents, int n, jk_select_plan_info* out) {
    JK_REQUIRE(cfg, "null argument");
    size_t slab[JK_MAX_DEPTH];
    return plan(*cfg, parents, n, out, slab);
}

extern "C" int jk_prior_select(jk_prior* p, const int32_t* parents, int n, void* workspace, size_t workspace_bytes,
                               jk_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    JK_REQUIRE(p, "null engine");
    JK_REQUIRE(p->t_host >= 0, "the last prefill stopped early (n_layers) and left later layers' caches unfilled: "
                               "there is no state to select from");
    jk_select_plan_info info;
    size_t slab[JK_MAX_DEPTH];
    int rc = plan(p->cfg, parents, n, &info, slab);
    if (rc) return rc;
    JK_REQUIRE(workspace_bytes >= info.workspace_bytes && (info.workspace_bytes == 0 || workspace),
               "workspace of %zu bytes, the selection stashes %d rows of %llu bytes: %llu needed", workspace_bytes,
               info.n_stash, (unsigned long long)info.row_bytes, (unsigned long long)info.workspace_bytes);
    JK_REQUIRE(((uintptr_t)workspace & 15) == 0, "workspace must be 16-byte aligned");
    if (info.n_copies == 0) return 0;
    SelectLaunch a;
    memset(&a, 0, sizeof(a));
    a.n_seg = 2 * p->cfg.depth;
    a.row_bytes = info.row_bytes;
    a.ws = (uint8_t*)workspace;
    unsigned long long chunks = 0, off = 0;
    for (int s = 0; s < a.n_seg; ++s) {
        a.first[s] = (unsigned)chunks;
        a.ws_off[s] = off;
        chunks += (slab[s >> 1] + kChunk - 1) / kChunk;
        off += slab[s >> 1];
    }
    JK_REQUIRE(chunks > 0 && chunks < (1ull << 31), "%llu chunks per row", chunks);
    a.first[a.n_seg] = (unsigned)chunks;
    int slot[JK_MAX_BATCH];
    for (int r = 0; r < n; ++r) slot[r] = -1;
    for (int i = 0; i < info.n_stash; ++i) slot[info.stash[i]] = i;
    int pairs = 0;
    if (info.n_stash) {          // stash: the rows that are read and overwritten, before anything is overwritten
        for (int i = 0; i < info.n_stash; ++i) { a.src[i] = (int8_t)info.stash[i]; a.dst[i] = (int8_t)(-1 - i); }
        select_copy_kernel<<<dim3((unsigned)chunks, info.n_stash), kSelThreads, 0, stream>>>(p->dev, a);
        JK_CHECK_CUDA(cudaGetLastError());
    }
    // copy: every source is a row that is not overwritten or a stash slot, so the launch's pairs are independent
    for (int b = 0; b < n; ++b) {
        if (parents[b] == b) continue;
        const int s = parents[b];
        a.src[pairs] = (int8_t)(slot[s] >= 0 ? -1 - slot[s] : s);
        a.dst[pairs] = (int8_t)b;
        pairs += 1;
    }
    select_copy_kernel<<<dim3((unsigned)chunks, pairs), kSelThreads, 0, stream>>>(p->dev, a);
    JK_CHECK_CUDA(cudaGetLastError());
    return 0;
}
