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
    return launch_attention(p, (cudaStream_t)stream);
}

}  // extern "C"
