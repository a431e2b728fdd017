// Attention core (see attention.cu).
#pragma once
#include "common.cuh"

namespace pb {

struct AttnParams {
    const __half* qkv;     // [B*P, 3E]: q | k_self | v_self
    const __half* ckv;     // [B, S_max, 2E]: k_cond | v_cond
    const int* kv_len;     // [slots] valid conditioning rows per cache slot (NULL: S_max)
    const int* kv_slot;    // [B] cache slot (sample block of ckv / entry of kv_len) each sample reads; NULL: slot = sample
    __half* out;           // [B*P, E]
    int B, P, S_max, E, nhead;
    int self_attn;         // keys = [self ; cond] (1) or cond only (0)
    float scale_log2;      // log2(e) / sqrt(head_dim)
    const float* attn_w;   // optional post-softmax weights for the last n_w keys ...
    int n_w;
    int w_batch;           // ... of samples [0, w_batch)
    int n_slots = 0;       // blocks of S_max rows in ckv (0: B)
    // Per-sample weights: attn_w is a table of rows w_ld floats apart.  Sample b < w_batch reads row w_row[b] (NULL: row b),
    // whose first w_len[row] entries (NULL: n_w) scale the last w_len[row] keys of its own [self ; cond] list; a length of 0
    // leaves the sample unweighted.  w_ld = 0 with w_len = NULL is the single vector of n_w entries shared by every sample.
    int w_ld = 0;
    const int* w_len = nullptr;
    const int* w_row = nullptr;
};

// Regional prompts, for samples b < mask_batch (the conditional rows).  Query q of sample b sees the conditioning of prompt k
// iff bit k of q_mask[b * P + q] is set: prompt 0 is the sample's own kv_slot[b], prompts 1..max_regions the cache slots
// region_slot[row * max_regions + k - 1] (-1: none), row = mask_row[b] (NULL: b), each read from its row 0 with its own
// kv_len.  Self keys stay visible to every query.  A separate kernel argument, so the plain instances keep their code.
struct AttnRegion {
    const uint8_t* q_mask;
    const int* region_slot;
    const int* mask_row;
    int max_regions;
    int mask_batch;
};

// Attention maps, for samples b < map_batch with map_row[b] >= 0 (NULL: row b): the instance writes, per head, the scaled scores
// s * scale_log2 of the sample's conditioning keys to scores [rows][nhead][P][S_max] (keys past kv_len untouched) and each query's
// m_run + log2(l_run) to lse2 [rows][nhead][P], so that exp2(score - lse2) is the softmax probability before attn_weights.  A
// separate kernel argument, so the plain instances keep their code.
struct AttnMapOut {
    float* scores;
    float* lse2;
    const int* map_row;
    int map_batch;
};

// The map row of sample b, or -1
__device__ __forceinline__ int attn_map_row(const AttnMapOut& mo, int b) {
    if (b >= mo.map_batch) return -1;
    return mo.map_row ? mo.map_row[b] : b;
}

// Prompt-to-prompt injection, for samples b < batch with src[b] >= 0: sample b replays sample src[b]'s attention probabilities.
// It loads Q and its self K from row src[b] and its conditioning K from slot kv_slot[src[b]], and its self V and conditioning V
// from its own row and slot; key counts come from its own kv_len (the caller keeps them equal to the source's).  attn_weights
// stay the sample's own.  With src[b] == b the instance computes what the instance without injection computes.  A separate
// kernel argument, so the plain instances keep their code.
struct AttnInject {
    const int* src;
    int batch;
};

// The sample whose queries and keys sample b uses: src[b], or b itself
__device__ __forceinline__ int attn_inj_src(const AttnInject& inj, int b) {
    if (b >= inj.batch) return b;
    const int a = inj.src[b];
    return a >= 0 ? a : b;
}

// Perturbed-attention guidance, for samples b < batch with bit `block` of block_mask[b] set (the launch's AttnBlock): the self
// part of every query's attention collapses onto the diagonal.  The self keys enter S, the running max and the denominator as
// usual, but their P (after attn_weights) is kept as a running self mass instead of entering P V, and mass * V_self[query] is
// added to O before the division; the conditioning keys' P is unchanged.  A perturbed sample is never regional, injected or
// a source.  A separate kernel argument, so the plain instances keep their code.
struct AttnPerturb {
    const uint64_t* block_mask;
    int batch;
    int block;
};

__device__ __forceinline__ bool attn_perturbed(const AttnPerturb& pt, int b) {
    return b < pt.batch && ((pt.block_mask[b] >> pt.block) & 1ull);
}

constexpr int ATT_MAX_REGIONS = 7;      // prompts 1..7: the mask bits above prompt 0's

// The key walk of a regional tile: segments of keys, each cut into 64-key chunks from its own first key.  Bit `bit` of a
// query's mask gates the segment's keys from `from` on (-1: none gated).
struct AttnSegs {
    int n;
    int first[ATT_MAX_REGIONS + 3];     // first chunk of segment i; first[n] = the tile's chunk count
    int slot[ATT_MAX_REGIONS + 2];      // cache slot the segment's conditioning keys come from
    int len[ATT_MAX_REGIONS + 2];       // keys
    int bit[ATT_MAX_REGIONS + 2];
    int from[ATT_MAX_REGIONS + 2];
};

// The OR of the masks of queries [q0, q0 + 64) of sample b (one warp; every lane gets it).  Samples past mask_batch see
// prompt 0 alone.
__device__ __forceinline__ uint32_t attn_tile_union(const AttnParams& p, const AttnRegion& rg, int b, int q0, int lane) {
    if (b >= rg.mask_batch) return 1u;
    uint32_t u = 0;
    for (int q = q0 + lane; q < q0 + 64 && q < p.P; q += 32) u |= rg.q_mask[(int64_t)b * p.P + q];
    return __reduce_or_sync(0xffffffffu, u);
}

// The mask of query row `row` of sample b (rows past P: every prompt, their output is never stored).
__device__ __forceinline__ uint32_t attn_row_mask(const AttnParams& p, const AttnRegion& rg, int b, int row) {
    if (b >= rg.mask_batch) return 1u;
    return row < p.P ? rg.q_mask[(int64_t)b * p.P + row] : 0xffu;
}

// One thread: the segments of a tile whose queries' masks OR to u.  concat_self: the self keys and prompt 0 form one segment
// (the mma.sync kernel's [self ; cond] walk, prompt 0 gated from key n_self on), otherwise the self keys are a segment of their
// own.  A prompt outside u gets no segment, so no chunk of it is loaded.
__device__ __forceinline__ void attn_build_segs(const AttnParams& p, const AttnRegion& rg, int b, uint32_t u, bool concat_self, AttnSegs& s) {
    const int n_self = p.self_attn ? p.P : 0;
    int n = 0, c = 0;
    auto add = [&](int slot, int len, int bit, int from) {
        s.first[n] = c; s.slot[n] = slot; s.len[n] = len; s.bit[n] = bit; s.from[n] = from;
        c += (len + 63) / 64;
        ++n;
    };
    const int slot0 = p.kv_slot ? p.kv_slot[b] : b;
    const int len0 = (u & 1u) ? (p.kv_len ? p.kv_len[slot0] : p.S_max) : 0;
    if (concat_self) {
        add(slot0, n_self + len0, 0, n_self);
    } else {
        if (n_self > 0) add(-1, n_self, -1, 0);
        if (u & 1u) add(slot0, len0, 0, 0);
    }
    if (b < rg.mask_batch && rg.region_slot) {
        const int row = rg.mask_row ? rg.mask_row[b] : b;
        for (int k = 1; k <= rg.max_regions && k <= ATT_MAX_REGIONS; ++k) {
            if (!((u >> k) & 1u)) continue;
            const int sl = rg.region_slot[(int64_t)row * rg.max_regions + k - 1];
            if (sl >= 0) add(sl, p.kv_len ? p.kv_len[sl] : p.S_max, k, 0);
        }
    }
    s.first[n] = c;
    s.n = n;
}

// The weight row of sample b and its length (0: unweighted), per the table layout above.
__device__ __forceinline__ int attn_weight_row(const AttnParams& p, int b, const float*& w) {
    if (p.attn_w == nullptr || b >= p.w_batch) return 0;
    const int row = p.w_row ? p.w_row[b] : b;
    w = p.attn_w + (int64_t)row * p.w_ld;
    return p.w_len ? p.w_len[row] : p.n_w;
}

// Dispatch: the wgmma + TMA kernel (attention_wg.cu) for head_dim 80, the mma.sync kernel (attention.cu) for other head dims
// (rg: the regional table, or NULL for the plain instances)
// (mo: the map outputs, or NULL.  With rg too, a map row's keys are its prompt 0's; its queries should all see prompt 0 alone.)
// (inj: the injection table, or NULL.  With rg too, only samples whose queries all see prompt 0 alone may be injected or be
// sources: an injected sample's prompt 0 keys come from its source's slot, further prompts' from their own.)
// (pt: the perturbation table, or NULL: the _perturb instances, with every combination of rg, mo and inj for the other rows.)
int launch_attention(const AttnParams& p, cudaStream_t st, const AttnRegion* rg = nullptr, const AttnMapOut* mo = nullptr,
                     const AttnInject* inj = nullptr, const AttnPerturb* pt = nullptr);
int launch_attention_wgmma(const AttnParams& p, cudaStream_t st, const AttnRegion* rg = nullptr, const AttnMapOut* mo = nullptr,
                           const AttnInject* inj = nullptr, const AttnPerturb* pt = nullptr);      // 0 launched, 1 error, -1 shape not handled
// Attention maps (ops.cu): acc [rows][acc_ld][acc_pos] += (1/nhead) * sum over heads h in ascending order of
// w_s * exp2(score - lse2) at columns [acc_off, acc_off + P), for every map row of p's batch and every conditioning key s < kv_len
int launch_attention_maps_accumulate(const AttnParams& p, const AttnMapOut& mo, float* acc, int acc_ld, int acc_pos, int acc_off,
                                     cudaStream_t st);
// maps [rows][S][h][w] = scale * sum over levels l, ascending, of acc[row][s][off_l + (y / (patch << l)) * gw_l + x / (patch << l)],
// off_l = sum of the grids (h / patch >> k) * (w / patch >> k) of the levels k < l
int launch_attention_maps_finalize(const float* acc, int rows, int acc_ld, int acc_pos, int S, int h, int w, int patch, int n_levels,
                                   float scale, float* maps, cudaStream_t st);
// Every AttnBlock level's position masks from token masks (ops.cu, regional_masks)
int launch_regional_masks(const uint8_t* tok_mask, const int* mask_row, int batch, int h, int w, int patch, int n_levels,
                          uint8_t* out, cudaStream_t st);

}  // namespace pb
