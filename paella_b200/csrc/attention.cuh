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
};

// Dispatch: the wgmma + TMA kernel (attention_wg.cu) for head_dim 80, the mma.sync kernel (attention.cu) for other head dims
int launch_attention(const AttnParams& p, cudaStream_t st);
int launch_attention_wgmma(const AttnParams& p, cudaStream_t st);      // 0 launched, 1 error, -1 shape not handled

}  // namespace pb
