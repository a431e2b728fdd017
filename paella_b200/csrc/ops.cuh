// Memory-bound kernels of the denoiser / codec (LayerNorm, depthwise conv, GRN, FiLM table, gathers, layout).
// All activations are channels-last.  See ops.cu for the reference lines each one replaces.
#pragma once
#include "common.cuh"

namespace pb {

// in_mapper + PixelUnshuffle: tokens [B,H,W] i64 -> fp16 [B*(H/ps)*(W/ps), c_in*ps*ps] (channel = c*ps*ps + dy*ps + dx)
int launch_embed_tokens(const int64_t* tokens, const float* emb, int num_labels, int c_in, int B, int H, int W, int ps,
                        __half* out, cudaStream_t st);

// LayerNorm over the last dim (eps 1e-6, no affine), optional scalar affine y*scale+shift, fp32 in.
// Exactly one of out16 / out32 is non-null.  rows x C, C % 4 == 0.  mean_out (optional): fp32 [rows] row means.
int launch_ln_rows(const float* x, int64_t rows, int C, float scale, float shift, __half* out16, float* out32,
                   cudaStream_t st, float* mean_out = nullptr);

// LN2d + 2x2 patchify: x fp32 [B,h,w,c] -> fp16 [B*(h/2)*(w/2), 4c] with column = (dy*2+dx)*c + ch
int launch_ln_patchify2(const float* x, int B, int h, int w, int c, __half* out, cudaStream_t st);

// ResBlock front: depthwise kxk conv (zero pad k/2; optional [x,skip] 2-channel groups) + bias + LN -> fp16 [M,c]
// w_packed: fp32 [k*k][per][c] (per = 1, or 2 with skip), bias fp32 [c]
// wrap (optional, DEVICE uint8): sample b wraps around on the axes of wrap[b < n_base ? b : b - n_base] (bit 0 x, bit 1 y);
// NULL launches the zero-padding kernels
int launch_dwconv_ln(const float* x, const float* skip, const float* w_packed, const float* bias, int B, int h, int w,
                     int c, int k, __half* out, cudaStream_t st, const uint8_t* wrap = nullptr, int n_base = 0);

// codec ResBlock front in one pass (ref/src/vqgan.py:36-40; see ops.cu): x' = x + g2*(dw3x3(reppad(LN(x)(1+g0)+g1)) + bias) -> x_out
// (a buffer other than x), a16 = fp16(LN(x')(1+g3)+g4).  gam = the block's gammas on the HOST; stats_scratch: B*h*w float2.
// wrap (optional, DEVICE uint8 [B]): circular instead of replication padding on the axes of wrap[b] (bit 0 x, bit 1 y)
bool vq_front_fused_ok(int c, int h, int w);
int launch_vq_front_fused(const float* x, int B, int h, int w, int c, const float* w9, const float* bias, const float* gam,
                          float2* stats_scratch, float* x_out, __half* a16, cudaStream_t st, const uint8_t* wrap = nullptr);

// GlobalResponseNorm: h[b,p,n] = h*(1 + gamma[n]*Gx[b,n]/(mean_n Gx + 1e-6)) + beta[n], Gx = sqrt(sq[b,n]) (2^-24 fixed point);
// zeroes all B*zero_per_sample entries of sq_next (the other buffer of a ping-pong pair) for the next block.
// scale_scratch: fp32 [B, N] (the per-sample multipliers, written by the first of the two launches)
int launch_grn_fused(__half* h, int B, int P, int N, const uint64_t* sq, uint64_t* sq_next, int zero_per_sample, const float* gamma,
                     const float* beta, float* scale_scratch, cudaStream_t st);

// gen_r_embedding: r [B] -> [B, c_r]
int launch_r_embed(const float* r, int B, int c_r, float* out, cudaStream_t st);
// all TimestepBlock mappers at once: out[b, j] = bias[j] + sum_i r_embed[b,i] * W[j,i]; W [total, c_r]
int launch_film_table(const float* r_embed, int B, int c_r, const float* W, const float* bias, int total, float* out,
                      cudaStream_t st);
// standalone FiLM: x[m,n] = x*(1+a[b,n]) + s[b,n]
int launch_film_apply(float* x, int64_t M, int N, int P, const float* film, int64_t film_ld, int64_t film_off,
                      cudaStream_t st);

int launch_cast_f16(const float* x, int64_t n, __half* out, cudaStream_t st);
int launch_silu_cast_f16(const float* x, int64_t n, __half* out, cudaStream_t st);
// fp32 NHWC [B,h,w,c] -> fp16 [B,h+2,w+2,c] with a one-position border: circular copies on the axes wrap[b] (DEVICE uint8 [B];
// bit 0 x, bit 1 y) wraps, zeros elsewhere (the ConvTranspose2d input of a tiled decode)
int launch_pad_cast_f16(const float* x, int B, int h, int w, int c, const uint8_t* wrap, __half* out, cudaStream_t st);
// out[i] = fp16(a[i]*wa + b[i]*wb)   (b may be null)
int launch_mix_cast_f16(const float* a, const float* b, float wa, float wb, int64_t n, __half* out, cudaStream_t st);
// the same mix with per-sample weights: element e uses (wa, wb) = (w[3 s], w[3 s + 1]), s = e / per (w: DEVICE [samples][3])
int launch_mix_cast_rows_f16(const float* a, const float* b, const float* w, int64_t per, int64_t n, __half* out, cudaStream_t st);
// the fp16 cast of whole samples of `per` elements into n_blocks packed blocks: block j < n_list is sample samples[j] of a,
// block j >= n_list is sample batch + samples[j - n_list] (samples: DEVICE int32 [n_list]); per % 4 == 0
int launch_gather_cast_f16(const float* a, const int* samples, int n_list, int n_blocks, int batch, int64_t per, __half* out,
                           cudaStream_t st);
// resample_logits_kernel<1> (mode 1, argmax) or resample_quant_kernel (mode 2) over `batch` packed samples of logits whose
// output sample is map[b] (DEVICE int32 [batch]): params row and token row map[b] (rng.cu)
int launch_resample_mapped(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw, const float* params,
                           const int* map, int mode, const float* codebook, int c_latent, int64_t* out, cudaStream_t st);

// tail rows: sample n_base + i of `base` (per bytes per sample) becomes a copy of sample src[i] (src: DEVICE int32 [n_tail])
int launch_replicate_rows(void* base, int64_t per, int n_base, const int* src, int n_tail, cudaStream_t st);
// guidance prompts, in place: per composed sample y, rows[y][0..ld) (DEVICE int32: c, u, then term samples, -1 = none) and
// coef[y][0..ld) (DEVICE fp32); sample c becomes fmaf(f_c, a_c, f_u*a_u), then fmaf(f_j, a_j, .) per term.  per % 4 == 0
int launch_guidance_mix(float* features, int64_t per, const int* rows, const float* coef, int n_composed, int ld, cudaStream_t st);

// [B, C, HW] <-> [B, HW, C] fp32
int launch_nchw_to_nhwc(const float* in, int B, int C, int HW, float* out, cudaStream_t st);
int launch_nhwc_to_nchw(const float* in, int B, int C, int HW, float* out, cudaStream_t st);

}  // namespace pb
