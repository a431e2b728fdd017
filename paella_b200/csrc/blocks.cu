// Block-level entry points of the C ABI: the kernels a stand-alone `ResBlock`, `AttnBlock`, `Attention2D`,
// `FeedForwardBlock`, `TimestepBlock`, `LayerNorm2d` or `GlobalResponseNorm` (ref/src/modules.py:7-106) is composed
// of when it is called outside a `Paella` (inside one, paella_model.cu runs the same kernels from its plan).
// The two kernels defined here exist only for that surface (general eps / affine LayerNorm, fp32 GRN); everything
// else forwards to the launchers the model executor uses.
#include "attention.cuh"
#include "ops.cuh"
#include "paella_b200.h"

namespace pb {

// LayerNorm over the last dim with arbitrary eps and optional per-channel affine (nn.LayerNorm semantics)
__global__ void __launch_bounds__(256) ln_affine_kernel(const float* __restrict__ x, int64_t rows, int C, float eps,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        float* __restrict__ out32, __half* __restrict__ out16) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const float* xr = x + row * C;
    float s = 0.f;
    for (int i = lane; i < C; i += 32) s += xr[i];
    const float mean = warp_sum(s) / C;
    float q = 0.f;
    for (int i = lane; i < C; i += 32) { const float d = xr[i] - mean; q = fmaf(d, d, q); }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / C + eps);
    for (int i = lane; i < C; i += 32) {
        float y = (xr[i] - mean) * rstd;
        if (gamma) y *= gamma[i];
        if (beta) y += beta[i];
        if (out16) out16[row * C + i] = __float2half_rn(y);
        else out32[row * C + i] = y;
    }
}

// GlobalResponseNorm on fp32 [B, P, N] (ref/src/modules.py:30-40): stat[b,n] = sqrt(sum_p x^2)
__global__ void __launch_bounds__(256) grn_f32_stat_kernel(const float* __restrict__ x, int P, int N, float* __restrict__ stat) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * 256 + threadIdx.x;
    if (n >= N) return;
    const float* xb = x + (int64_t)b * P * N + n;
    float s = 0.f;
    for (int p = 0; p < P; ++p) { const float v = xb[(int64_t)p * N]; s = fmaf(v, v, s); }
    stat[(int64_t)b * N + n] = sqrtf(s);
}

__global__ void __launch_bounds__(256) grn_f32_apply_kernel(const float* __restrict__ x, int P, int N, const float* __restrict__ stat,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            float* __restrict__ out) {
    const int b = blockIdx.y;
    const float* sb = stat + (int64_t)b * N;
    float s = 0.f;
    for (int i = threadIdx.x; i < N; i += 256) s += sb[i];
    __shared__ float red[8];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += red[i];
    const float inv = 1.0f / (tot / N + 1e-6f);
    const int64_t base = (int64_t)b * P * N;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < (int64_t)P * N; i += (int64_t)gridDim.x * 256) {
        const int n = (int)(i % N);
        const float v = x[base + i];
        out[base + i] = fmaf(gamma[n], v * (sb[n] * inv), beta[n]) + v;
    }
}

}  // namespace pb

using namespace pb;

extern "C" {

int pb200_layernorm(const float* x, int64_t rows, int c, float eps, const float* weight, const float* bias, float* out32,
                    void* out16, void* stream) {
    PB_CHECK(x != nullptr && rows >= 0 && c > 0, "layernorm: bad arguments");
    PB_CHECK((out32 != nullptr) != (out16 != nullptr), "layernorm: exactly one output");
    if (rows == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (eps == 1e-6f && !weight && !bias && c % 4 == 0)      // the denoiser's own LayerNorm2d: the executor's kernel
        return launch_ln_rows(x, rows, c, 1.0f, 0.0f, reinterpret_cast<__half*>(out16), out32, st);
    ln_affine_kernel<<<ceil_div(rows, 8), 256, 0, st>>>(x, rows, c, eps, weight, bias, out32, reinterpret_cast<__half*>(out16));
    PB_LAUNCH_CHECK();
    return 0;
}

int pb200_nchw_to_nhwc(const float* in, int batch, int c, int hw, float* out, void* stream) {
    PB_CHECK(in && out, "nchw_to_nhwc: null pointer");
    return launch_nchw_to_nhwc(in, batch, c, hw, out, (cudaStream_t)stream);
}

int pb200_nhwc_to_nchw(const float* in, int batch, int c, int hw, float* out, void* stream) {
    PB_CHECK(in && out, "nhwc_to_nchw: null pointer");
    return launch_nhwc_to_nchw(in, batch, c, hw, out, (cudaStream_t)stream);
}

int pb200_cast_f16(const float* x, int64_t n, int silu, void* out16, void* stream) {
    PB_CHECK(x && out16, "cast_f16: null pointer");
    if (n == 0) return 0;
    return silu ? launch_silu_cast_f16(x, n, reinterpret_cast<__half*>(out16), (cudaStream_t)stream)
                : launch_cast_f16(x, n, reinterpret_cast<__half*>(out16), (cudaStream_t)stream);
}

int pb200_dwconv_ln(const float* x, const float* skip, const float* w_packed, const float* bias, int batch, int h, int w,
                    int c, int k, void* out16, void* stream) {
    PB_CHECK(x && w_packed && bias && out16, "dwconv_ln: null pointer");
    if (batch == 0) return 0;
    return launch_dwconv_ln(x, skip, w_packed, bias, batch, h, w, c, k, reinterpret_cast<__half*>(out16), (cudaStream_t)stream);
}

int pb200_dwconv_ln_tiled(const float* x, const float* skip, const float* w_packed, const float* bias, int batch, int h, int w,
                          int c, int k, const uint8_t* wrap, void* out16, void* stream) {
    PB_CHECK(x && w_packed && bias && out16, "dwconv_ln: null pointer");
    if (batch == 0) return 0;
    return launch_dwconv_ln(x, skip, w_packed, bias, batch, h, w, c, k, reinterpret_cast<__half*>(out16), (cudaStream_t)stream,
                            wrap, batch);
}

int pb200_grn_f16(void* h16, int batch, int rows_per_sample, int n, const uint64_t* sqsum, uint64_t* sqsum_next,
                  int zero_per_sample, const float* gamma, const float* beta, float* scale_scratch, void* stream) {
    PB_CHECK(h16 && sqsum && sqsum_next && gamma && beta && scale_scratch, "grn_f16: null pointer");
    PB_CHECK(sqsum != sqsum_next, "grn_f16: the statistic being read and the one being zeroed must differ");
    return launch_grn_fused(reinterpret_cast<__half*>(h16), batch, rows_per_sample, n, sqsum, sqsum_next, zero_per_sample, gamma, beta,
                            scale_scratch, (cudaStream_t)stream);
}

int pb200_grn_f32(const float* x, int batch, int rows_per_sample, int n, const float* gamma, const float* beta, float* stat,
                  float* out, void* stream) {
    PB_CHECK(x && gamma && beta && stat && out, "grn_f32: null pointer");
    if (batch == 0 || rows_per_sample == 0) return 0;
    PB_CHECK(batch <= 65535, "grn_f32: batch too large");
    cudaStream_t st = (cudaStream_t)stream;
    grn_f32_stat_kernel<<<dim3(ceil_div(n, 256), batch), 256, 0, st>>>(x, rows_per_sample, n, stat);
    PB_LAUNCH_CHECK();
    const int64_t per = (int64_t)rows_per_sample * n;
    const int gx = (int)(per / 256 / 8 > 0 ? (per / 256 / 8 > 1024 ? 1024 : per / 256 / 8) : 1);
    grn_f32_apply_kernel<<<dim3(gx, batch), 256, 0, st>>>(x, rows_per_sample, n, stat, gamma, beta, out);
    PB_LAUNCH_CHECK();
    return 0;
}

int pb200_film_apply(float* x, int64_t rows, int n, int rows_per_sample, const float* film, int64_t film_ld, int64_t film_off,
                     void* stream) {
    PB_CHECK(x && film && rows_per_sample > 0, "film_apply: bad arguments");
    if (rows == 0) return 0;
    return launch_film_apply(x, rows, n, rows_per_sample, film, film_ld, film_off, (cudaStream_t)stream);
}

// ---- executor kernels exposed for testing: thin forwards to the launchers paella_model.cu runs from its plan.  Every
// refusal happens before anything is enqueued.
int pb200_embed_tokens(const int64_t* tokens, const float* emb, int num_labels, int c_in, int batch, int h, int w, int patch,
                       void* out16, void* stream) {
    PB_CHECK(tokens && emb && out16, "embed_tokens: null pointer");
    PB_CHECK(num_labels > 0 && c_in > 0 && patch > 0 && batch >= 0 && h >= 0 && w >= 0, "embed_tokens: bad arguments");
    if ((int64_t)batch * h * w == 0) return 0;
    return launch_embed_tokens(tokens, emb, num_labels, c_in, batch, h, w, patch, reinterpret_cast<__half*>(out16),
                               (cudaStream_t)stream);
}

int pb200_ln_rows(const float* x, int64_t rows, int c, float scale, float shift, void* out16, float* out32, float* mean_out,
                  void* stream) {
    PB_CHECK(x != nullptr && rows >= 0 && c > 0, "ln_rows: bad arguments");
    return launch_ln_rows(x, rows, c, scale, shift, reinterpret_cast<__half*>(out16), out32, (cudaStream_t)stream, mean_out);
}

int pb200_ln_patchify2(const float* x, int batch, int h, int w, int c, void* out16, void* stream) {
    PB_CHECK(x && out16, "ln_patchify2: null pointer");
    PB_CHECK(batch >= 0 && h >= 0 && w >= 0 && c > 0, "ln_patchify2: bad arguments");
    if ((int64_t)batch * h * w == 0) return 0;
    return launch_ln_patchify2(x, batch, h, w, c, reinterpret_cast<__half*>(out16), (cudaStream_t)stream);
}

int pb200_film_table(const float* r_embed, int batch, int c_r, const float* weight, const float* bias, int total, float* out,
                     void* stream) {
    PB_CHECK(r_embed && weight && bias && out, "film_table: null pointer");
    PB_CHECK(batch >= 0 && c_r > 0 && total >= 0, "film_table: bad arguments");
    if (batch == 0) return 0;
    return launch_film_table(r_embed, batch, c_r, weight, bias, total, out, (cudaStream_t)stream);
}

int pb200_mix_cast_f16(const float* a, const float* b, float wa, float wb, int64_t n, void* out16, void* stream) {
    PB_CHECK(a && out16 && n >= 0, "mix_cast: bad arguments");
    return launch_mix_cast_f16(a, b, wa, wb, n, reinterpret_cast<__half*>(out16), (cudaStream_t)stream);
}

int pb200_mix_cast_rows_f16(const float* a, const float* b, const float* w, int64_t per, int64_t n, void* out16, void* stream) {
    PB_CHECK(a && b && w && out16 && n >= 0, "mix_cast_rows: bad arguments");
    return launch_mix_cast_rows_f16(a, b, w, per, n, reinterpret_cast<__half*>(out16), (cudaStream_t)stream);
}

int pb200_pad_cast_f16(const float* x, int batch, int h, int w, int c, const uint8_t* wrap, void* out16, void* stream) {
    PB_CHECK(x && out16, "pad_cast: null pointer");
    PB_CHECK(batch >= 0 && h > 0 && w > 0 && c > 0, "pad_cast: bad arguments");
    return launch_pad_cast_f16(x, batch, h, w, c, wrap, reinterpret_cast<__half*>(out16), (cudaStream_t)stream);
}

int pb200_gather_cast_f16(const float* a, const int* samples, int n_list, int n_blocks, int batch, int64_t per, void* out16,
                          void* stream) {
    PB_CHECK(a && samples && out16, "gather_cast: null pointer");
    PB_CHECK(n_list >= 0 && n_blocks >= 0 && batch >= 0 && per >= 0, "gather_cast: bad arguments");
    return launch_gather_cast_f16(a, samples, n_list, n_blocks, batch, per, reinterpret_cast<__half*>(out16), (cudaStream_t)stream);
}

int pb200_replicate_rows(void* base, int64_t per, int n_base, const int* src, int n_tail, void* stream) {
    PB_CHECK(base && src, "replicate_rows: null pointer");
    PB_CHECK(per >= 0 && n_base >= 0 && n_tail >= 0, "replicate_rows: bad arguments");
    return launch_replicate_rows(base, per, n_base, src, n_tail, (cudaStream_t)stream);
}

int pb200_regional_masks(const uint8_t* tok_mask, const int* mask_row, int batch, int h, int w, int patch, int n_levels, uint8_t* out,
                         void* stream) {
    PB_CHECK(tok_mask && out, "regional_masks: null pointer");
    PB_CHECK(batch >= 0 && patch > 0 && n_levels > 0 && n_levels <= PB200_MAX_LEVELS && h >= (patch << (n_levels - 1)) &&
                 w >= (patch << (n_levels - 1)),
             "regional_masks: %d levels of patch %d on a %dx%d grid", n_levels, patch, h, w);
    return launch_regional_masks(tok_mask, mask_row, batch, h, w, patch, n_levels, out, (cudaStream_t)stream);
}

int pb200_guidance_mix(float* features, int64_t per, const int* rows, const float* coef, int n_composed, int ld, void* stream) {
    PB_CHECK(features && rows && coef, "guidance_mix: null pointer");
    PB_CHECK(per >= 0 && n_composed >= 0, "guidance_mix: bad arguments");
    return launch_guidance_mix(features, per, rows, coef, n_composed, ld, (cudaStream_t)stream);
}

int pb200_dwconv_ln_pairs(const float* x, const float* skip, const float* w_packed, const float* bias, int batch, int h, int w,
                          int c, int k, const uint8_t* wrap, int n_base, void* out16, void* stream) {
    PB_CHECK(x && w_packed && bias && out16 && wrap, "dwconv_ln: null pointer");
    PB_CHECK(n_base > 0 && n_base <= batch && batch <= 2 * n_base, "dwconv_ln: %d samples with %d wrap codes", batch, n_base);
    return launch_dwconv_ln(x, skip, w_packed, bias, batch, h, w, c, k, reinterpret_cast<__half*>(out16), (cudaStream_t)stream,
                            wrap, n_base);
}

int pb200_attention(const void* qkv16, const void* ckv16, const int* kv_len, void* out16, int batch, int positions, int s_max,
                    int embed, int nhead, int self_attn, const float* attn_weights, int n_weights, int weighted_batch,
                    void* stream) {
    return pb200_attention_slots(qkv16, ckv16, kv_len, nullptr, 0, out16, batch, positions, s_max, embed, nhead, self_attn,
                                 attn_weights, n_weights, 0, nullptr, nullptr, weighted_batch, stream);
}

int pb200_attention_slots(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                          int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                          int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                          void* stream) {
    return pb200_attention_regional(qkv16, ckv16, kv_len, kv_slot, n_slots, out16, batch, positions, s_max, embed, nhead, self_attn,
                                    attn_weights, n_weights, weights_ld, weights_len, weights_row, weighted_batch, nullptr, nullptr,
                                    nullptr, 0, 0, stream);
}

int pb200_attention_regional(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                             int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                             int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                             const uint8_t* q_mask, const int* region_slot, const int* mask_row, int max_regions, int mask_batch,
                             void* stream) {
    PB_CHECK(qkv16 && out16 && (ckv16 || s_max == 0), "attention: null pointer");
    PB_CHECK(self_attn || s_max > 0, "attention: no keys");
    PB_CHECK(n_slots >= 0 && weights_ld >= 0, "attention: negative slot count or weight stride");
    AttnParams p{};
    p.qkv = reinterpret_cast<const __half*>(qkv16);
    p.ckv = reinterpret_cast<const __half*>(ckv16 ? ckv16 : qkv16);
    p.kv_len = kv_len;
    p.kv_slot = kv_slot;
    p.n_slots = n_slots;
    p.out = reinterpret_cast<__half*>(out16);
    p.B = batch; p.P = positions; p.S_max = s_max; p.E = embed; p.nhead = nhead;
    p.self_attn = self_attn;
    p.scale_log2 = 1.4426950408889634f / sqrtf((float)(embed / (nhead > 0 ? nhead : 1)));
    p.attn_w = attn_weights; p.n_w = attn_weights ? n_weights : 0; p.w_batch = weighted_batch;
    p.w_ld = weights_ld; p.w_len = weights_len; p.w_row = weights_row;
    if (q_mask == nullptr) return launch_attention(p, (cudaStream_t)stream);
    PB_CHECK(max_regions >= 0 && max_regions <= ATT_MAX_REGIONS, "attention: max_regions=%d (0..%d)", max_regions, ATT_MAX_REGIONS);
    PB_CHECK(mask_batch >= 0 && mask_batch <= batch, "attention: mask_batch=%d for %d samples", mask_batch, batch);
    PB_CHECK(region_slot != nullptr || max_regions == 0, "attention: regional prompts need region_slot");
    const AttnRegion rg{q_mask, region_slot, mask_row, max_regions, mask_batch};
    return launch_attention(p, (cudaStream_t)stream, &rg);
}

int pb200_attention_maps(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                         int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                         int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                         float* scores, float* lse2, const int* map_row, int map_batch, void* stream) {
    PB_CHECK(qkv16 && out16 && (ckv16 || s_max == 0), "attention: null pointer");
    PB_CHECK(self_attn || s_max > 0, "attention: no keys");
    PB_CHECK(n_slots >= 0 && weights_ld >= 0, "attention: negative slot count or weight stride");
    PB_CHECK(map_batch >= 0 && map_batch <= batch && (map_batch == 0 || (scores && lse2)), "attention: map_batch=%d for %d samples",
             map_batch, batch);
    AttnParams p{};
    p.qkv = reinterpret_cast<const __half*>(qkv16);
    p.ckv = reinterpret_cast<const __half*>(ckv16 ? ckv16 : qkv16);
    p.kv_len = kv_len;
    p.kv_slot = kv_slot;
    p.n_slots = n_slots;
    p.out = reinterpret_cast<__half*>(out16);
    p.B = batch; p.P = positions; p.S_max = s_max; p.E = embed; p.nhead = nhead;
    p.self_attn = self_attn;
    p.scale_log2 = 1.4426950408889634f / sqrtf((float)(embed / (nhead > 0 ? nhead : 1)));
    p.attn_w = attn_weights; p.n_w = attn_weights ? n_weights : 0; p.w_batch = weighted_batch;
    p.w_ld = weights_ld; p.w_len = weights_len; p.w_row = weights_row;
    const AttnMapOut mo{scores, lse2, map_row, map_batch};
    return launch_attention(p, (cudaStream_t)stream, nullptr, &mo);
}

int pb200_attention_inject(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                           int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                           int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                           const uint8_t* q_mask, const int* region_slot, const int* mask_row, int max_regions, int mask_batch,
                           float* scores, float* lse2, const int* map_row, int map_batch, const int* inj_src, int inj_batch,
                           void* stream) {
    PB_CHECK(qkv16 && out16 && (ckv16 || s_max == 0), "attention: null pointer");
    PB_CHECK(self_attn || s_max > 0, "attention: no keys");
    PB_CHECK(n_slots >= 0 && weights_ld >= 0, "attention: negative slot count or weight stride");
    PB_CHECK(q_mask == nullptr || (mask_batch >= 0 && mask_batch <= batch && max_regions >= 0 && max_regions <= ATT_MAX_REGIONS &&
                                   (region_slot != nullptr || max_regions == 0)),
             "attention: regional table (mask_batch=%d, max_regions=%d) for %d samples", mask_batch, max_regions, batch);
    PB_CHECK(map_batch >= 0 && map_batch <= batch && (map_batch == 0 || (scores && lse2)), "attention: map_batch=%d for %d samples",
             map_batch, batch);
    PB_CHECK(inj_batch >= 0 && inj_batch <= batch && (inj_batch == 0 || inj_src), "attention: inj_batch=%d for %d samples", inj_batch,
             batch);
    AttnParams p{};
    p.qkv = reinterpret_cast<const __half*>(qkv16);
    p.ckv = reinterpret_cast<const __half*>(ckv16 ? ckv16 : qkv16);
    p.kv_len = kv_len;
    p.kv_slot = kv_slot;
    p.n_slots = n_slots;
    p.out = reinterpret_cast<__half*>(out16);
    p.B = batch; p.P = positions; p.S_max = s_max; p.E = embed; p.nhead = nhead;
    p.self_attn = self_attn;
    p.scale_log2 = 1.4426950408889634f / sqrtf((float)(embed / (nhead > 0 ? nhead : 1)));
    p.attn_w = attn_weights; p.n_w = attn_weights ? n_weights : 0; p.w_batch = weighted_batch;
    p.w_ld = weights_ld; p.w_len = weights_len; p.w_row = weights_row;
    const AttnRegion rg{q_mask, region_slot, mask_row, max_regions, mask_batch};
    const AttnMapOut mo{scores, lse2, map_row, map_batch};
    const AttnInject inj{inj_src, inj_batch};
    return launch_attention(p, (cudaStream_t)stream, q_mask ? &rg : nullptr, map_batch > 0 ? &mo : nullptr, inj_batch > 0 ? &inj : nullptr);
}

int pb200_attention_perturb(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                            int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                            int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                            const uint8_t* q_mask, const int* region_slot, const int* mask_row, int max_regions, int mask_batch,
                            float* scores, float* lse2, const int* map_row, int map_batch, const int* inj_src, int inj_batch,
                            const uint64_t* pag_mask, int pag_batch, int pag_block, void* stream) {
    PB_CHECK(pag_batch >= 0 && pag_batch <= batch && (pag_batch == 0 || pag_mask) && pag_block >= 0 && pag_block < 64,
             "attention: pag_batch=%d for %d samples, block %d", pag_batch, batch, pag_block);
    if (pag_batch == 0)
        return pb200_attention_inject(qkv16, ckv16, kv_len, kv_slot, n_slots, out16, batch, positions, s_max, embed, nhead, self_attn,
                                      attn_weights, n_weights, weights_ld, weights_len, weights_row, weighted_batch, q_mask, region_slot,
                                      mask_row, max_regions, mask_batch, scores, lse2, map_row, map_batch, inj_src, inj_batch, stream);
    PB_CHECK(qkv16 && out16 && (ckv16 || s_max == 0), "attention: null pointer");
    PB_CHECK(self_attn || s_max > 0, "attention: no keys");
    PB_CHECK(n_slots >= 0 && weights_ld >= 0, "attention: negative slot count or weight stride");
    PB_CHECK(q_mask == nullptr || (mask_batch >= 0 && mask_batch <= batch && max_regions >= 0 && max_regions <= ATT_MAX_REGIONS &&
                                   (region_slot != nullptr || max_regions == 0)),
             "attention: regional table (mask_batch=%d, max_regions=%d) for %d samples", mask_batch, max_regions, batch);
    PB_CHECK(map_batch >= 0 && map_batch <= batch && (map_batch == 0 || (scores && lse2)), "attention: map_batch=%d for %d samples",
             map_batch, batch);
    PB_CHECK(inj_batch >= 0 && inj_batch <= batch && (inj_batch == 0 || inj_src), "attention: inj_batch=%d for %d samples", inj_batch,
             batch);
    AttnParams p{};
    p.qkv = reinterpret_cast<const __half*>(qkv16);
    p.ckv = reinterpret_cast<const __half*>(ckv16 ? ckv16 : qkv16);
    p.kv_len = kv_len;
    p.kv_slot = kv_slot;
    p.n_slots = n_slots;
    p.out = reinterpret_cast<__half*>(out16);
    p.B = batch; p.P = positions; p.S_max = s_max; p.E = embed; p.nhead = nhead;
    p.self_attn = self_attn;
    p.scale_log2 = 1.4426950408889634f / sqrtf((float)(embed / (nhead > 0 ? nhead : 1)));
    p.attn_w = attn_weights; p.n_w = attn_weights ? n_weights : 0; p.w_batch = weighted_batch;
    p.w_ld = weights_ld; p.w_len = weights_len; p.w_row = weights_row;
    const AttnRegion rg{q_mask, region_slot, mask_row, max_regions, mask_batch};
    const AttnMapOut mo{scores, lse2, map_row, map_batch};
    const AttnInject inj{inj_src, inj_batch};
    const AttnPerturb pt{pag_mask, pag_batch, pag_block};
    return launch_attention(p, (cudaStream_t)stream, q_mask ? &rg : nullptr, map_batch > 0 ? &mo : nullptr, inj_batch > 0 ? &inj : nullptr,
                            &pt);
}

}  // extern "C"
