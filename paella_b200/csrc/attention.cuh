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

// The weight row of sample b and its length (0: unweighted), per the table layout above.
__device__ __forceinline__ int attn_weight_row(const AttnParams& p, int b, const float*& w) {
    if (p.attn_w == nullptr || b >= p.w_batch) return 0;
    const int row = p.w_row ? p.w_row[b] : b;
    w = p.attn_w + (int64_t)row * p.w_ld;
    return p.w_len ? p.w_len[row] : p.n_w;
}

// Dispatch: the wgmma + TMA kernel (attention_wg.cu) for head_dim 80, the mma.sync kernel (attention.cu) for other head dims
int launch_attention(const AttnParams& p, cudaStream_t st);
int launch_attention_wgmma(const AttnParams& p, cudaStream_t st);      // 0 launched, 1 error, -1 shape not handled

}  // namespace pb
