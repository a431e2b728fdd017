/* paella_b200 — C ABI of the Paella hot path, native to the H100 (sm_90a).
 *
 * The reference (dome272/Paella @ e1ab72b) has no FFI layer: its boundary is the
 * Python class surface (SURVEY.md §8b).  This header is the C ABI the Python
 * mirror in paella_b200/ binds with ctypes; each entry point names the reference
 * code it replaces.  Conventions:
 *   - every pointer is a DEVICE pointer unless the name says `host`;
 *   - no function allocates or frees caller memory; scratch comes in as `workspace`;
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*), no hidden syncs;
 *   - return 0 on success, non-zero on error with the text in pb200_last_error();
 *   - there is NO CPU fallback anywhere.
 * Layout: "NCHW"/"NHWC" as named; activations inside the library are channels-last.
 */
#ifndef PAELLA_B200_H
#define PAELLA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB200_ABI_VERSION 4      /* 4: GEMM A-operand scaling and the two always-0 pb200_gemm_plan outputs removed.
                                    * Bumped when an entry point changes or goes away; new entry points keep it. */

const char* pb200_last_error(void);
int pb200_abi_version(void);
/* multiprocessor count / max threads per SM of the current device (they fix PyTorch's Philox launch policy). */
int pb200_device_info(int* sm_count, int* max_threads_per_sm);

/* Measurement hooks used by bench.py: number of kernel launches the library has made so far, and optional
 * CUDA-event bracketing of every launch by kernel family (report: JSON {family: {launches, ms, work}},
 * work = algorithmic FLOPs for GEMM-shaped kernels, bytes otherwise). */
long long pb200_launch_count(void);
int pb200_profile_enable(int on);
int pb200_profile_report(char* buf, long long cap);

/* ------------------------------------------------------------------------------------------
 * Random streams and the resample step.  `seed`/`offset` are the (seed, philox offset) of the
 * torch CUDA generator BEFORE the op; each op consumes pb200_philox_offset_increment(numel)
 * offsets, exactly like the torch op it replaces, so a caller that advances the torch
 * generator by that amount stays on the reference's random stream.
 * ------------------------------------------------------------------------------------------ */
/* philox offsets one distribution kernel over `numel` elements consumes
 * (ATen/native/cuda/DistributionTemplates.h:50-62). */
int64_t pb200_philox_offset_increment(int64_t numel);

/* torch.randint(0, num_labels, size) -> int64   [ref/src/utils.py:37] */
int pb200_randint(int64_t* out, int64_t numel, int64_t num_labels, uint64_t seed, uint64_t offset, void* stream);

/* torch.rand(numel) fp32 in [0,1)               [the draw inside ref/src/modules.py:279] */
int pb200_rand(float* out, int64_t numel, uint64_t seed, uint64_t offset, void* stream);

/* torch.multinomial(p, 1)[:, 0] for p fp32 [rows, k] row-major; BIT-EXACT with torch given the
 * same generator state (argmax_k p/q, q = Tensor.exponential_(1))   [ref/src/utils.py:49-50] */
int pb200_multinomial(const float* p, int64_t rows, int64_t k, uint64_t seed, uint64_t offset, int64_t* out,
                      void* stream);

/* The whole resample expression of ref/src/utils.py:45-50 on reference-layout logits:
 *   l = logits_c*cfg + logits_u*(1-cfg)   (logits_u may be NULL: no guidance)
 *   p = softmax(l * (1/temperature), dim=1);  token = multinomial(p)
 * logits_*: fp32 NCHW [B, K, HW].  out: int64 [B, HW].
 * mode 0 = multinomial, 1 = argmax of logits (notebook `mode='argmax'`).
 * Same arithmetic as torch op-by-op except the softmax denominator's summation order. */
int pb200_resample_logits(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw,
                          double cfg, double temperature, int mode, uint64_t seed, uint64_t offset, int64_t* out,
                          void* stream);

/* `quant` sampling mode (notebook cell 3; ref/src_distributed/train.py:155-156): e = softmax(l/T) @ codebook,
 * token = nearest code of e.  logits as above; codebook fp32 [k, c_latent]; no random draw. */
int pb200_resample_quant(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw, double cfg,
                         double temperature, const float* codebook, int c_latent, int64_t* out, void* stream);

/* Per-sample sampling parameters.  params: DEVICE float [batch][3] = (cfg_b, 1 - cfg_b, 1 / temperature_b) as the fp32
 * constants the scalar entry points derive from their double arguments: (float)cfg, (float)(1.0 - cfg) and
 * 1.0f / (float)temperature.  Sample b is computed with row b exactly as the scalar call on (cfg_b, temperature_b) computes it;
 * the cfg columns are ignored where there is no guidance (logits_u == NULL, cfg_on == 0). */

/* pb200_resample_logits with per-sample (cfg, 1 - cfg, 1/T) in one launch over the batch; the draw is the scalar call's. */
int pb200_resample_logits_params(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw,
                                 const float* params, int mode, uint64_t seed, uint64_t offset, int64_t* out, void* stream);

/* pb200_resample_quant with per-sample (cfg, 1 - cfg, 1/T) in one launch over the batch. */
int pb200_resample_quant_params(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw,
                                const float* params, const float* codebook, int c_latent, int64_t* out, void* stream);

/* Paella.add_noise(x, t, random_x=...)            [ref/src/modules.py:277-283]
 *   mask = (rand_like(x.float()) <= t[:,None,None]); x*(1-mask) + random_x*mask
 * x, random_x, out: int64 [B, HW]; t: fp32 [B]; mask_out: int64 [B, HW] or NULL.
 * random_x == NULL -> randint_like(x, 0, num_labels) drawn AFTER the mask draw (second offset block). */
int pb200_add_noise(const int64_t* x, const int64_t* random_x, const float* t, int64_t batch, int64_t hw,
                    int64_t num_labels, uint64_t seed, uint64_t offset, int64_t* out, int64_t* mask_out,
                    void* stream);
/* pb200_add_noise restricted to a token region: inpainting / outpainting from source tokens.  With the reference's
 * explicit-mask add_noise [ref/src/modules.py:277-283, ref/utils/modules.py:282-288] and the init_x of sample_distributed
 * [ref/src_distributed/utils.py:97-126] it computes, element for element,
 *   m   = (rand_like(x.float()) <= t[:,None,None]) & region
 *   out = where(region, x*(1-m) + random_x*m, src)          mask_out = m
 * src: int64 [B, HW] (the kept tokens), region: uint8 [B, HW] (nonzero = generated), indexed like random_x; both NULL is
 * pb200_add_noise, which is this call.  The draws are those of pb200_add_noise whatever the region.  A sample with t < 0 is
 * never renoised, so such a launch only composites: it needs no fresh Philox offset. */
int pb200_add_noise_region(const int64_t* x, const int64_t* random_x, const int64_t* src, const uint8_t* region, const float* t,
                           int64_t batch, int64_t hw, int64_t num_labels, uint64_t seed, uint64_t offset, int64_t* out,
                           int64_t* mask_out, void* stream);

/* One random stream per sample, in ONE launch over the batch (a list of per-sample torch.Generators).  seed_offset: DEVICE
 * uint64 [batch][2] = (seed, philox offset) of sample b's generator before the draw, offsets multiples of 4.  Sample b draws
 * exactly what the batch-1 entry point draws on (seed, offset) = seed_offset[b] (torch's launch policy for numel = hw), and
 * each generator is to be advanced by pb200_philox_offset_increment(hw) per draw.  hw <= 2^29, batch <= 65535.
 * slot: int32 [batch] or NULL (identity): sample b's row of `out` (and of random_x) is row slot[b] of that buffer. */
int pb200_randint_per_sample(int64_t* out, const int* slot, int64_t batch, int64_t hw, int64_t num_labels,
                             const uint64_t* seed_offset, void* stream);
/* pb200_add_noise per sample: x int64 [batch, hw] and mask_out (or NULL) by sample; t fp32 [batch], and a sample with t < 0
 * keeps its tokens; random_x (by slot) or NULL -> randint_like drawn after the mask draw, as pb200_add_noise does. */
int pb200_add_noise_per_sample(const int64_t* x, const int64_t* random_x, const int* slot, const float* t, int64_t batch,
                               int64_t hw, int64_t num_labels, const uint64_t* seed_offset, int64_t* out, int64_t* mask_out,
                               void* stream);
/* pb200_add_noise_per_sample restricted to a token region, as pb200_add_noise_region [ref/src/modules.py:277-283,
 * ref/utils/modules.py:282-288]: src and region are indexed by slot like random_x and out.  Both NULL is
 * pb200_add_noise_per_sample, which is this call. */
int pb200_add_noise_region_per_sample(const int64_t* x, const int64_t* random_x, const int64_t* src, const uint8_t* region,
                                      const int* slot, const float* t, int64_t batch, int64_t hw, int64_t num_labels,
                                      const uint64_t* seed_offset, int64_t* out, int64_t* mask_out, void* stream);
/* Confidence-guided renoise: replaces pb200_add_noise_region's random mask [ref/src/modules.py:277-283] by each sample's
 * least likely tokens.  logp: fp32 [batch, hw], the step's log-probability of each drawn token (pb200_paella_token_logprob);
 * t: fp32 [batch] next noise levels; tau: fp32 [batch] choice temperatures.  For sample b with tau[b] >= 0 and N candidate tokens
 * (those inside region, all without one): u_j is the uniform pb200_add_noise_region draws for the token (same stream and element,
 * so the offset consumed is the same), k_j = logp_j + (tau t) g_j with g_j = -logf(-logf(u_j)) (each operation rounded in fp32),
 * and the n = floor(fp32(t * N)) candidates with the smallest keys are renoised, ties to the lower token index; a NaN key ranks
 * below every other.  A sample with tau[b] < 0 is pb200_add_noise_region's own rule (u <= t), bit for bit, and one with t < 0
 * keeps its tokens.  out = where(region, where(mask, random_x, x), src); mask_out (or NULL) = the renoised tokens.  random_x is
 * required; src and region are both NULL or both set.  hw <= 32768 (the selection keeps a sample's keys in shared memory). */
int pb200_renoise_confidence(const int64_t* x, const int64_t* random_x, const int64_t* src, const uint8_t* region, const float* logp,
                             const float* t, const float* tau, int64_t batch, int64_t hw, uint64_t seed, uint64_t offset,
                             int64_t* out, int64_t* mask_out, void* stream);
/* pb200_renoise_confidence on per-sample streams, replacing pb200_add_noise_region_per_sample: sample b draws on
 * seed_offset[b]; slot (int32 [batch] or NULL = identity) places its rows of random_x, src, region and out at slot[b]; x, logp
 * and mask_out are by sample. */
int pb200_renoise_confidence_per_sample(const int64_t* x, const int64_t* random_x, const int64_t* src, const uint8_t* region,
                                        const int* slot, const float* logp, const float* t, const float* tau, int64_t batch,
                                        int64_t hw, const uint64_t* seed_offset, int64_t* out, int64_t* mask_out, void* stream);
/* out[b] = pool[slot[b]] for rows of hw int64 tokens (b < batch): a step batch gathered from a token pool. */
int pb200_gather_rows(const int64_t* pool, const int* slot, int64_t batch, int64_t hw, int64_t* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Vector quantiser (torchtools.nn.VectorQuantize; call sites ref/src/vqgan.py:94,104).
 * ------------------------------------------------------------------------------------------ */
/* nearest code (first minimum of |c|^2+|x|^2-2x.c, fp32 fma chain — oracle/vq_nearest.c).
 * x: fp32 [n, c] (channels-last vectors); codebook fp32 [k, c], c <= 8; idx: int64 [n]. */
int pb200_vq_nearest(const float* x, int64_t n, int c, const float* codebook, int k, int64_t* idx, void* stream);
/* idx2vq: out[n, c] = codebook[idx[n]] (channels-last). */
int pb200_vq_gather(const int64_t* idx, int64_t n, const float* codebook, int k, int c, float* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Tensor-core GEMM (wgmma, TMA-fed, register accumulators): C[M,N] = A[M,K] . W[N,K]^T (+epilogue)
 * A, W: fp16 row-major (K contiguous), K % 8 == 0.  Used by every 1x1-conv / Linear of the path;
 * exported for unit tests.
 * ------------------------------------------------------------------------------------------ */
enum pb200_epilogue {
    PB200_EPI_F16 = 0,        /* out fp16 [M,ldo]   = acc + bias                                        */
    PB200_EPI_F32 = 1,        /* out fp32 [M,ldo]   = acc + bias                                        */
    PB200_EPI_GELU_F16 = 2,   /* out fp16 = gelu_erf(acc + bias); sqsum[row/rows_per_sample, n] += out^2 */
    PB200_EPI_RESID_F32 = 3,  /* out fp32 = ((acc + bias)*alpha + resid) [* (1+film_a) + film_b]         */
    PB200_EPI_UNPATCH_F32 = 4,/* out fp32 NHWC [B,2h,2w,cout]: col=(dy,dx,co), row=(b,y,x); bias[col]    */
    PB200_EPI_NCHW_F32 = 5,   /* out fp32 [B, N, hw]: row=(b,p) -> out[b][n][p]; acc + bias              */
    /* LayerNorm folded across two GEMMs (the AttnBlock's pre-norm, ref/src/modules.py:78): the producer also emits
     * the fp16 copy of its output row and the row statistics, the consumer multiplies the UN-normalised fp16 rows and
     * normalises in its epilogue:  LN(x) W^T = rstd * (x W^T - mean * rowsum(W)). */
    PB200_EPI_RESID_LN_F32 = 6, /* RESID_F32 + out16[M,ldo] = fp16(out - s); ln_stat[row] += (sum (out-s), sum (out-s)^2),
                                 * s = ln_shift[row] (0 if NULL).  LayerNorm is invariant under a per-row shift, so any s
                                 * is exact; an s near the row mean keeps the fp16 rounding of the copy relative to the row's
                                 * SPREAD instead of its offset (the executor passes the mean the previous AttnBlock saw). */
    PB200_EPI_F16_LN = 7,      /* out fp16 = rstd[row]*(acc - mean'[row]*ln_wsum[n]) + bias, (mean', rstd) of the shifted
                                 * rows from ln_stat; if ln_mean_out: ln_mean_out[row] = ln_shift[row] + mean' (true mean) */
    PB200_EPI_RESID_LN_INV_F32 = 8 /* RESID_LN_F32 with batch-invariant statistics: each 32-column chunk's row sums are
                                 * rounded to the ln_stat fixed point on their own and added as integers, so ln_stat does
                                 * not depend on the tile width (which the planner picks from M) or the CTA order */
};

typedef struct pb200_gemm_epilogue {
    int mode;                  /* enum pb200_epilogue */
    const float* bias;         /* [N] or NULL */
    void* out;
    int64_t ldo;               /* leading dimension of out in elements (F16/F32/GELU/RESID) */
    const float* resid;        /* RESID: fp32 [M, ldr] (may alias out) */
    int64_t ldr;
    float alpha;               /* RESID: scale on (acc+bias); 1.0 for the denoiser */
    uint64_t* sqsum;           /* GELU: [M/rows_per_sample, N] sum of out^2 in 2^-24 fixed point (integer atomics:
                                  order-independent, hence run-to-run deterministic), or NULL */
    int rows_per_sample;       /* GELU/RESID(film)/NCHW: rows of one sample */
    const float* film;         /* RESID: fp32 [B, film_ld]: a = film[b, film_off + n], b = film[b, film_off + N + n]; or NULL */
    int64_t film_ld;
    int64_t film_off;
    int remap_in, remap_out;   /* F16/F32: out_row = (row/remap_in)*remap_out + row%remap_in; 0 = identity */
    int up_h, up_w, up_cout;   /* UNPATCH: coarse grid and output channels */
    void* out16;               /* RESID_LN: fp16 [M, ldo] copy of out */
    int64_t* ln_stat;          /* RESID_LN (accumulated, caller zeroes) / F16_LN (read): [M][2] = (sum x * 2^20, sum x^2 * 2^16)
                                  over the ln_c columns of a row, fixed point (integer atomics: order-independent) */
    const float* ln_wsum;      /* F16_LN: [N] row sums of the fp16 weight matrix */
    int ln_c;                  /* F16_LN: number of columns the statistics cover (= K of this GEMM) */
    const float* ln_shift;     /* RESID_LN / F16_LN: fp32 [M] per-row shift the producer subtracted, or NULL (= 0) */
    float* ln_mean_out;        /* F16_LN: fp32 [M] true row mean (shift + mean of the shifted row), or NULL */
} pb200_gemm_epilogue;

int pb200_gemm_f16(const void* a, int64_t lda, const void* w, int64_t ldw, int64_t m, int64_t n, int64_t k,
                   const pb200_gemm_epilogue* epi, void* stream);
/* Host-side tile plan pb200_gemm_f16 would use for an [m,k] x [n,k]^T problem on `sm_count` multiprocessors (0 = the
 * current device, or 132 without one): BLOCK_N (one CTA per tile, every tile BLOCK_N wide).  Pure arithmetic, no device
 * work. */
int pb200_gemm_plan(int64_t m, int64_t n, int64_t k, int sm_count, int* block_n);

/* ------------------------------------------------------------------------------------------
 * Block-level kernels: what the reference's building-block modules (ref/src/modules.py:7-106)
 * run when they are called on their own, outside a Paella (inside one the model executor below
 * launches the same kernels from its plan).  Activations are channels-last rows [batch*positions, c]
 * unless named NCHW; "16" pointers are fp16.
 * ------------------------------------------------------------------------------------------ */
/* nn.LayerNorm over the last dim: y = (x-mean)/sqrt(var+eps) [*weight + bias]; exactly one of out32/out16.
 * LayerNorm2d = this between the two layout changes below   [ref/src/modules.py:22-27] */
int pb200_layernorm(const float* x, int64_t rows, int c, float eps, const float* weight, const float* bias, float* out32,
                    void* out16, void* stream);
/* x.permute(0,2,3,1) / x.permute(0,3,1,2) on fp32 [batch, c, hw] <-> [batch, hw, c]   [ref/src/modules.py:27,58-61] */
int pb200_nchw_to_nhwc(const float* in, int batch, int c, int hw, float* out, void* stream);
int pb200_nhwc_to_nchw(const float* in, int batch, int c, int hw, float* out, void* stream);
/* fp32 -> fp16 GEMM operand, optionally through SiLU (AttnBlock.kv_mapper[0])   [ref/src/modules.py:71-74] */
int pb200_cast_f16(const float* x, int64_t n, int silu, void* out16, void* stream);
/* ResBlock front: depthwise k x k conv over cat[x, skip] (groups = c, zero padding k/2) + bias + LayerNorm2d(no
 * affine, eps 1e-6) -> fp16 [batch*h*w, c].  x fp32 NHWC [batch,h,w,c]; skip NHWC [batch,h,w,c] or NULL;
 * w_packed fp32 [k*k][per][c] (per = 2 with skip: concatenated input channels 2g, 2g+1 feed output g)
 * [ref/src/modules.py:46-47,57-58] */
int pb200_dwconv_ln(const float* x, const float* skip, const float* w_packed, const float* bias, int batch, int h, int w,
                    int c, int k, void* out16, void* stream);
/* pb200_dwconv_ln with per-sample circular padding: sample b wraps on the axes of wrap[b] (DEVICE uint8 [batch]; bit 0 x,
 * bit 1 y), zero padding elsewhere.  wrap = NULL is pb200_dwconv_ln. */
int pb200_dwconv_ln_tiled(const float* x, const float* skip, const float* w_packed, const float* bias, int batch, int h, int w,
                          int c, int k, const uint8_t* wrap, void* out16, void* stream);
/* GlobalResponseNorm in place on the fp16 hidden [batch, rows_per_sample, n] of a PB200_EPI_GELU_F16 GEMM whose
 * epilogue accumulated sqsum (2^-24 fixed point); zeroes zero_per_sample entries per sample of sqsum_next;
 * scale_scratch = caller-owned fp32 [batch, n] (the per-sample multipliers 1 + gamma * Nx, written then read)
 * [ref/src/modules.py:30-40] */
int pb200_grn_f16(void* h16, int batch, int rows_per_sample, int n, const uint64_t* sqsum, uint64_t* sqsum_next,
                  int zero_per_sample, const float* gamma, const float* beta, float* scale_scratch, void* stream);
/* GlobalResponseNorm.forward on an fp32 NHWC tensor [batch, rows_per_sample, n]; stat = scratch [batch, n]
 * [ref/src/modules.py:37-40] */
int pb200_grn_f32(const float* x, int batch, int rows_per_sample, int n, const float* gamma, const float* beta, float* stat,
                  float* out, void* stream);
/* TimestepBlock: x[r, j] = x*(1 + film[r/rows_per_sample, film_off + j]) + film[.., film_off + n + j] in place
 * [ref/src/modules.py:104-106] */
int pb200_film_apply(float* x, int64_t rows, int n, int rows_per_sample, const float* film, int64_t film_ld, int64_t film_off,
                     void* stream);
/* ------------------------------------------------------------------------------------------
 * Executor kernels exposed for testing: the launchers the model executor below runs from its plan,
 * with every argument it passes them, so that each kernel can be checked on its own against a
 * high-precision reference.  A refusal returns nonzero (pb200_last_error) with nothing enqueued.
 * ------------------------------------------------------------------------------------------ */
/* in_mapper (Embedding + LayerNorm, eps 1e-6) + PixelUnshuffle(patch): tokens int64 [batch, h, w] (clamped to
 * [0, num_labels)), emb fp32 [num_labels, c_in] -> fp16 [batch*(h/patch)*(w/patch), c_in*patch^2], column c*patch^2 +
 * dy*patch + dx; c_in*patch^2 <= 3072   [ref/src/modules.py:126-131,271] */
int pb200_embed_tokens(const int64_t* tokens, const float* emb, int num_labels, int c_in, int batch, int h, int w, int patch,
                       void* out16, void* stream);
/* LayerNorm over rows of c % 4 == 0 fp32 values (eps 1e-6) with a scalar affine: y = (x-mean)*rstd*scale + shift into exactly
 * one of out16 / out32 (out32 may be x: in place); mean_out (optional) fp32 [rows] = the row means */
int pb200_ln_rows(const float* x, int64_t rows, int c, float scale, float shift, void* out16, float* out32, float* mean_out,
                  void* stream);
/* LayerNorm2d + the im2col of Conv2d(k=2, s=2): x fp32 NHWC [batch, h, w, c] (h, w even, c % 4 == 0) -> fp16
 * [batch*(h/2)*(w/2), 4c], column (dy*2 + dx)*c + ch   [ref/src/modules.py:153-156] */
int pb200_ln_patchify2(const float* x, int batch, int h, int w, int c, void* out16, void* stream);
/* every TimestepBlock mapper at once: out[b, j] = bias[j] + sum_i r_embed[b, i] * weight[j, i]; weight fp32 [total, c_r]
 * [ref/src/modules.py:99-106] */
int pb200_film_table(const float* r_embed, int batch, int c_r, const float* weight, const float* bias, int total, float* out,
                     void* stream);
/* out16[i] = fp16(a[i]*wa + b[i]*wb) (b NULL: a[i]*wa), i < n */
int pb200_mix_cast_f16(const float* a, const float* b, float wa, float wb, int64_t n, void* out16, void* stream);
/* the same mix with per-sample weights: element e of sample s = e / per uses (w[3s], w[3s+1]) (w DEVICE fp32 [samples][3]) */
int pb200_mix_cast_rows_f16(const float* a, const float* b, const float* w, int64_t per, int64_t n, void* out16, void* stream);
/* fp32 NHWC [batch, h, w, c] -> fp16 [batch, h+2, w+2, c] with a one-position border: circular copies on the axes wrap[b]
 * (DEVICE uint8 [batch]; bit 0 x, bit 1 y) wraps, zeros on the others; c % 4 == 0 */
int pb200_pad_cast_f16(const float* x, int batch, int h, int w, int c, const uint8_t* wrap, void* out16, void* stream);
/* fp16 cast of whole samples of `per` fp32 elements into n_blocks packed blocks: block j < n_list is sample samples[j] of a,
 * block j >= n_list is sample batch + samples[j - n_list] (samples DEVICE int32 [n_list]); per % 4 == 0, n_blocks <= 2*n_list */
int pb200_gather_cast_f16(const float* a, const int* samples, int n_list, int n_blocks, int batch, int64_t per, void* out16,
                          void* stream);
/* sample n_base + i of base (per bytes per sample, base 16-byte aligned) becomes a copy of sample src[i] (DEVICE int32 [n_tail]) */
int pb200_replicate_rows(void* base, int64_t per, int n_base, const int* src, int n_tail, void* stream);
/* per-level regional masks: level l of out holds uint8 [batch][(h/s)*(w/s)], s = patch << l, at offset batch * (sum of the
 * earlier levels' sizes); each value is the OR of its s x s footprint of token-mask row mask_row[b] (NULL: b) of tok_mask
 * (DEVICE uint8 [rows, h*w]) */
int pb200_regional_masks(const uint8_t* tok_mask, const int* mask_row, int batch, int h, int w, int patch, int n_levels, uint8_t* out,
                         void* stream);
/* pb200_paella_guidance_mix on `per` fp32 elements per sample (per % 4 == 0, features 16-byte aligned), without a model */
int pb200_guidance_mix(float* features, int64_t per, const int* rows, const float* coef, int n_composed, int ld, void* stream);
/* pb200_dwconv_ln_tiled on a CFG batch: sample b reads wrap[b < n_base ? b : b - n_base] (n_base <= batch <= 2*n_base) */
int pb200_dwconv_ln_pairs(const float* x, const float* skip, const float* w_packed, const float* bias, int batch, int h, int w,
                          int c, int k, const uint8_t* wrap, int n_base, void* out16, void* stream);
/* Attention core of nn.MultiheadAttention / CustomMultiheadAttention after the in-projection:
 * qkv16 [batch*positions, 3*embed] = q | k_self | v_self, ckv16 [batch, s_max, 2*embed] = k_cond | v_cond
 * (kv_len[batch] valid rows, NULL = s_max); keys = [self ; cond] if self_attn else cond; optional post-softmax
 * attn_weights on the last n_weights keys of samples [0, weighted_batch); out16 [batch*positions, embed]
 * [ref/src/modules.py:12-19, ref/utils/alter_attention.py:19-36] */
int pb200_attention(const void* qkv16, const void* ckv16, const int* kv_len, void* out16, int batch, int positions, int s_max,
                    int embed, int nhead, int self_attn, const float* attn_weights, int n_weights, int weighted_batch,
                    void* stream);
/* pb200_attention with shared conditioning slots and a per-sample weight table (pb200_attention is this call with
 * kv_slot = NULL, n_slots = 0, weights_ld = 0, weights_len = weights_row = NULL):
 *   kv_slot      int32 [batch]: the block of s_max rows of ckv16 (and the entry of kv_len) sample b reads, or NULL: block b;
 *   n_slots      blocks in ckv16 and entries in kv_len (0: batch);
 *   attn_weights fp32 table of rows weights_ld floats apart; sample b < weighted_batch reads row weights_row[b] (NULL: row b),
 *                whose first weights_len[row] entries (NULL: n_weights) scale the last weights_len[row] keys of its own
 *                [self ; cond] list; a length of 0 leaves the sample unweighted.  weights_ld = 0 with weights_len = NULL is
 *                one vector of n_weights entries shared by every sample. */
int pb200_attention_slots(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                          int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                          int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                          void* stream);
/* pb200_attention_slots with regional prompts, for samples b < mask_batch:
 *   q_mask       uint8 [mask_batch][positions]: bit k of query q's byte set = it sees the conditioning of prompt k;
 *   region_slot  int32 [rows][max_regions]: the block of ckv16 (and entry of kv_len) of prompts 1..max_regions, -1 = none;
 *   mask_row     int32 [mask_batch]: the region_slot row sample b reads, or NULL: row b;
 *   max_regions  0..7.
 * Prompt 0 is sample b's own block kv_slot[b].  A query attends, in one softmax, to every self key and to the conditioning
 * keys of each prompt whose bit it has; a query must have at least one bit (or self_attn).  A tile of 64 queries loads no
 * key of a prompt none of them sees.  Samples b >= mask_batch attend as in pb200_attention_slots, and a query whose byte is
 * 1 (prompt 0 alone) gets the same bits as there.  attn_weights apply to [self ; prompt 0] and must not be combined with
 * regions on one sample.  [ref/src/modules.py:7-19 with a boolean attn_mask on nn.MultiheadAttention] */
int pb200_attention_regional(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                             int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                             int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                             const uint8_t* q_mask, const int* region_slot, const int* mask_row, int max_regions, int mask_batch,
                             void* stream);
/* pb200_attention_slots with attention maps, for samples b < map_batch whose map row mr = map_row[b] (NULL: b) is >= 0:
 *   scores  fp32 [rows][nhead][positions][s_max]: query q's scaled score s * log2(e) / sqrt(head_dim) on each of the sample's
 *           conditioning keys j < kv_len (entries past kv_len are not written);
 *   lse2    fp32 [rows][nhead][positions]: query q's log2 of the softmax denominator over [self ; cond] keys, in the same units.
 * exp2(score - lse2) is then the softmax probability of the key before attn_weights.  out16 gets the bits of
 * pb200_attention_slots on the same inputs.  [ref/utils/alter_attention.py:4-43 with need_weights=True] */
int pb200_attention_maps(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                         int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                         int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                         float* scores, float* lse2, const int* map_row, int map_batch, void* stream);
/* Prompt-to-prompt injection: pb200_attention_regional (q_mask NULL: no regions) with optional attention maps
 * (pb200_attention_maps; map_batch 0: none), where sample b < inj_batch with a = inj_src[b] >= 0 (DEVICE int32 [inj_batch], -1:
 * none) replays sample a's attention probabilities:
 *   out[b] = (softmax(scale * Q_a [K_a,self ; K_a,cond]^T) * w_b) [V_b,self ; V_b,cond]
 * Q_a and K_a,self are sample a's rows of qkv16, K_a,cond its slot kv_slot[a]'s; the values, kv_len and the weights w_b are
 * sample b's own.  The caller keeps kv_len of b's and a's slots equal.  With q_mask, an injected sample and its source must see
 * prompt 0 alone at every query.  inj_src[b] == b gives the bits of the call without injection.  A map row of an injected
 * sample holds the replayed probabilities.  [prompt-to-prompt editing, Hertz et al. 2022, on ref/utils/alter_attention.py] */
int pb200_attention_inject(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                           int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                           int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                           const uint8_t* q_mask, const int* region_slot, const int* mask_row, int max_regions, int mask_batch,
                           float* scores, float* lse2, const int* map_row, int map_batch, const int* inj_src, int inj_batch,
                           void* stream);
/* Perturbed-attention guidance: pb200_attention_inject where sample b < pag_batch with bit pag_block of pag_mask[b] set (DEVICE
 * uint64 [pag_batch]) has the self part of its attention collapsed onto the diagonal:
 *   P = softmax(scale * q_p [K_self ; K_cond]^T) * w_b,   out[b, p] = (sum_{j in self} P_pj) V_self,p + sum_{k in cond} P_pk V_cond,k
 * The conditioning probabilities are unchanged; with no conditioning keys out[b, p] = V_self,p.  A perturbed sample is not
 * regional, injected or a source.  Every other sample gets the bits of pb200_attention_inject.  pag_batch = 0 is
 * pb200_attention_inject, the same launch.  [perturbed-attention guidance, Ahn et al. 2024, on ref/src/modules.py Attention2D] */
int pb200_attention_perturb(const void* qkv16, const void* ckv16, const int* kv_len, const int* kv_slot, int n_slots, void* out16,
                            int batch, int positions, int s_max, int embed, int nhead, int self_attn, const float* attn_weights,
                            int n_weights, int weights_ld, const int* weights_len, const int* weights_row, int weighted_batch,
                            const uint8_t* q_mask, const int* region_slot, const int* mask_row, int max_regions, int mask_batch,
                            float* scores, float* lse2, const int* map_row, int map_batch, const int* inj_src, int inj_batch,
                            const uint64_t* pag_mask, int pag_batch, int pag_block, void* stream);

/* ------------------------------------------------------------------------------------------
 * Denoiser (ref/src/modules.py:109-283, ref/utils/modules.py) as an opaque handle.
 * ------------------------------------------------------------------------------------------ */
#define PB200_MAX_LEVELS 4

typedef struct pb200_paella_config {   /* constructor kwargs of Paella, ref/src/modules.py:110-112 */
    int c_in, c_out, num_labels, c_r, patch_size, c_cond;
    int n_levels;
    int c_hidden[PB200_MAX_LEVELS];
    int nhead[PB200_MAX_LEVELS];
    int blocks[PB200_MAX_LEVELS];
    char level_config[PB200_MAX_LEVELS][8];   /* e.g. "CT", "CTA" */
    int clip_embd, byt5_embd, clip_seq_len, kernel_size, self_attn;
} pb200_paella_config;

typedef struct pb200_paella pb200_paella;     /* opaque */

/* Build the layer plan (host only).  Weights live in a caller-owned device blob of
 * pb200_paella_weight_bytes() bytes, filled by pb200_paella_load_param(); the blob is
 * position-independent, so one rank can fill it and broadcast it (NCCL) to the others. */
int pb200_paella_create(const pb200_paella_config* cfg, pb200_paella** out);
void pb200_paella_destroy(pb200_paella* m);
int64_t pb200_paella_weight_bytes(const pb200_paella* m);
int pb200_paella_bind_weights(pb200_paella* m, void* weight_blob);
/* number / names of the state-dict entries the plan consumes (reference key names). */
int pb200_paella_num_params(const pb200_paella* m);
const char* pb200_paella_param_name(const pb200_paella* m, int i);
int64_t pb200_paella_param_numel(const pb200_paella* m, int i);
/* convert one reference-layout fp32 parameter (device pointer) into the packed blob. */
int pb200_paella_load_param(pb200_paella* m, const char* name, const float* src, int64_t numel, void* stream);
/* Handle option (default 0).  on = 1: batch-invariant forward -- every sample's features are bit-identical whatever batch,
 * batch position, CFG pairing or GPU count it runs in (the folded LayerNorm's row statistics use
 * PB200_EPI_RESID_LN_INV_F32).  on = 0: the default arithmetic.  Set it before forwards are enqueued, not concurrently
 * with them: forwards already enqueued keep the mode they were enqueued with. */
int pb200_paella_set_batch_invariant(pb200_paella* m, int on);

/* conditioning for `batch` samples: byt5 fp32 [B, L, byt5_embd]; clip / clip_image fp32
 * [B, clip_embd] or NULL; n_clip_image images (list-valued clip_image, ref/utils/modules.py:228-235,
 * laid out [n_img, B, clip_embd]).  Sequence length S = L + clip_seq_len*(has_clip + n_clip_image). */
typedef struct pb200_cond {
    const float* byt5; int byt5_len;
    const float* clip;
    const float* clip_image; int n_clip_image;
} pb200_cond;

/* scratch sizes for a forward over `batch_total` samples on an H x W token grid whose
 * conditioning sequences are at most `s_max` long. */
int64_t pb200_paella_workspace_bytes(const pb200_paella* m, int batch_total, int h, int w, int s_max);
/* bytes of the per-call conditioning cache (c_embed + every AttnBlock's cond K/V). */
int64_t pb200_paella_cond_cache_bytes(const pb200_paella* m, int batch_total, int s_max);

/* gen_c_embeddings + every AttnBlock's kv_mapper and K/V projection of the conditioning rows
 * (x- and t-independent) for samples [batch_offset, batch_offset + batch) of the cache. */
int pb200_paella_prepare_cond(pb200_paella* m, const pb200_cond* cond, int batch, int batch_offset, int batch_total,
                              int s_max, void* cond_cache, void* workspace, int64_t workspace_bytes, void* stream);

/* gen_r_embedding: r fp32 [B] -> fp32 [B, c_r]   (ref/src/modules.py:212-221) */
int pb200_paella_r_embedding(const float* r, int batch, int c_r, float* out, void* stream);
/* gen_c_embeddings: -> fp32 [B, S, c_cond], S = byt5_len + clip_seq_len*(has_clip + n_clip_image)   (ref/src/modules.py:223-232) */
int pb200_paella_c_embeddings(pb200_paella* m, const pb200_cond* cond, int batch, float* out, void* workspace,
                              int64_t workspace_bytes, void* stream);

/* Paella.forward up to out_mapper's LayerNorm: tokens int64 [Bt,H,W], r fp32 [Bt] ->
 * features fp32 [Bt*H*W, c_out] (rows (b,y,x)).  attn_weights fp32 [n_attn_weights] or NULL scales
 * the last n key columns after the softmax for samples [0, attn_weights_batch)
 * (ref/utils/alter_attention.py:23-34; the notebook passes it on the conditional forward only).
 * cond_cache was prepared for cache_slots sample slots (the batch_total of pb200_paella_prepare_cond); kv_slot int32
 * [batch_total] names the slot each sample attends to (NULL: slot i for sample i, cache_slots == batch_total) -- samples
 * with identical conditioning, e.g. the unconditional half of a CFG batch, share one slot and its K/V is read once.
 * cfg_pairs = 1: the classifier-free-guidance batch of ref/src/utils.py:42-45 -- tokens [Bt/2,H,W] and r [Bt/2] are
 * given once, sample i + Bt/2 is sample i under the unconditional rows of the conditioning cache.  The blocks before
 * the first AttnBlock do not see the conditioning and are evaluated once per pair (identical arithmetic). */
int pb200_paella_features(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int cfg_pairs, int h, int w,
                          const void* cond_cache, int cache_slots, const int* kv_slot, int s_max, const float* attn_weights,
                          int n_attn_weights,
                          int attn_weights_batch, float* features, void* workspace, int64_t workspace_bytes,
                          void* stream);
/* pb200_paella_features with guidance for only some samples: tokens [Bc,H,W] and r [Bc], Bc = batch_total - n_pairs; sample
 * Bc + i (i < n_pairs) is sample i under its unconditional rows (kv_slot[Bc + i]).  n_pairs = batch_total / 2 is
 * cfg_pairs = 1, n_pairs = 0 is cfg_pairs = 0. */
int pb200_paella_features_pairs(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_pairs, int h,
                                int w, const void* cond_cache, int cache_slots, const int* kv_slot, int s_max,
                                const float* attn_weights, int n_attn_weights, int attn_weights_batch, float* features,
                                void* workspace, int64_t workspace_bytes, void* stream);
/* pb200_paella_features_pairs with one attn_weights vector per sample, so that samples whose prompts (and so whose
 * vectors) differ share one forward.  It replaces the per-call `attn_weights` of CustomMultiheadAttention.forward
 * (ref/utils/alter_attention.py:23-34), which the notebook's text-to-image cell builds from each prompt's ByT5 length.
 *   attn_w  fp32 table of rows w_ld floats apart (device memory), or NULL for no weights at all;
 *   w_len   int32 [rows]: the length of each row (0: the sample is unweighted), or NULL: every row has n_w entries;
 *   w_row   int32 [w_batch]: the row sample b reads, or NULL: row b;
 *   w_batch samples [0, w_batch) are weighted (the unconditional tail of a CFG batch is not, as in the reference).
 * Sample b scales, after the softmax and without renormalising, the last w_len[row] keys of its own [self ; cond] key list
 * in every AttnBlock.  Each length must not exceed the smallest key count that sample sees in any AttnBlock, where the
 * reference fails.  w_ld = 0 with w_len = NULL is the single vector of pb200_paella_features_pairs, which is this call. */
int pb200_paella_features_weighted(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_pairs, int h,
                                   int w, const void* cond_cache, int cache_slots, const int* kv_slot, int s_max,
                                   const float* attn_w, int n_w, int w_ld, const int* w_len, const int* w_row, int w_batch,
                                   float* features, void* workspace, int64_t workspace_bytes, void* stream);
/* pb200_paella_features_weighted with seamless tiling: wrap = DEVICE uint8 [batch_total - n_pairs], one byte per sample, bit 0
 * wraps x (left and right edges), bit 1 wraps y.  On a wrapped axis the ResBlocks' depthwise convolutions pad circularly
 * (Conv2d padding_mode='circular'); the unconditional row batch_total - n_pairs + i reads byte i.  Nothing else depends on
 * it.  wrap = NULL is pb200_paella_features_weighted, the same launches; a byte-0 sample gives the same bits either way. */
int pb200_paella_features_tiled(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_pairs, int h, int w,
                                const void* cond_cache, int cache_slots, const int* kv_slot, int s_max, const float* attn_w, int n_w,
                                int w_ld, const int* w_len, const int* w_row, int w_batch, const uint8_t* wrap, float* features,
                                void* workspace, int64_t workspace_bytes, void* stream);
/* pb200_paella_features_tiled with regional prompts on the conditional rows [0, batch_total - n_pairs):
 *   prompt_mask  DEVICE uint8 [rows][h*w] token masks: bit k (k >= 1) set = the token lies in region k, bit 0 = in no region;
 *   mask_row     DEVICE int32 [batch_total - n_pairs]: the prompt_mask / region_slot row of sample b, or NULL: row b;
 *   region_slot  DEVICE int32 [rows][max_regions]: the cache slot of prompt k >= 1 (projected like any conditioning), -1 = none;
 *   max_regions  0..7.
 * A position of an AttnBlock level (stride patch_size * 2^level tokens) carries the OR of its footprint's token masks and attends
 * to every self key and to the conditioning of each prompt it has a bit of, prompt 0 being the sample's own kv_slot (see
 * pb200_attention_regional).  The unconditional rows are never masked.  attn weights must not be set on a regional sample.
 * prompt_mask = NULL is pb200_paella_features_tiled, the same launches. */
int pb200_paella_features_regional(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_pairs, int h,
                                   int w, const void* cond_cache, int cache_slots, const int* kv_slot, int s_max, const float* attn_w,
                                   int n_w, int w_ld, const int* w_len, const int* w_row, int w_batch, const uint8_t* wrap,
                                   const uint8_t* prompt_mask, const int* mask_row, const int* region_slot, int max_regions,
                                   float* features, void* workspace, int64_t workspace_bytes, void* stream);
/* pb200_paella_features_regional with an arbitrary tail: the batch is [batch_total - n_tail base samples; n_tail tail rows], and
 * tail row batch_total - n_tail + i carries the tokens and r of base sample tail_src[i] (DEVICE int32 [n_tail], each in
 * [0, batch_total - n_tail)) under its own kv_slot entry.  The conditioning-free prefix (everything before the first AttnBlock)
 * runs once on the base samples and is gathered to the tail rows, so a tail row's features equal those of its source's tokens
 * and r run as an ordinary row with that K/V slot.  A sample may own several tail rows (guidance prompts: one conditional
 * forward per extra prompt); n_tail < batch_total.  A tail row reads its source's wrap byte, and is never masked (prompt_mask
 * covers the base rows only) nor weighted (attn weights cover rows [0, w_batch), w_batch <= batch_total - n_tail).
 * tail_src = NULL is [0, n_tail), the unconditional rows of a CFG batch: pb200_paella_features_regional, the same launches. */
int pb200_paella_features_tail(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_tail, int h, int w,
                               const void* cond_cache, int cache_slots, const int* kv_slot, int s_max, const float* attn_w, int n_w,
                               int w_ld, const int* w_len, const int* w_row, int w_batch, const uint8_t* wrap, const uint8_t* prompt_mask,
                               const int* mask_row, const int* region_slot, int max_regions, const int* tail_src, float* features,
                               void* workspace, int64_t workspace_bytes, void* stream);
/* Attention maps: pb200_paella_features_tail that also accumulates, for base samples b < map_batch whose map row
 * mr = map_row[b] (DEVICE int32 [map_batch], NULL: b) is >= 0, each AttnBlock's cross-attention map into
 *   map_acc  DEVICE fp32 [map_rows][map_len][n_pos], n_pos = the sum over levels l of (h / (patch << l)) * (w / (patch << l)),
 *            caller-owned and caller-zeroed:
 *            map_acc[mr][s][off_l + p] += (1 / nhead_l) * sum over heads of P[p, n_self + s], level l's block positions p at
 *            off_l (level 0 first), for every conditioning key s < min(kv_len, map_len).
 * P is the softmax over [self ; cond] keys times the sample's attn weights (post-softmax, not renormalised), so the sums are the
 * probabilities ref/utils/alter_attention.py returns with need_weights=True.  Each AttnBlock then runs the maps instance of the
 * attention kernel and an accumulate kernel; features are bit-identical to the call without maps, and each map row's sums depend
 * on its sample alone (no atomics).  The workspace must hold pb200_paella_workspace_bytes + pb200_paella_maps_workspace_bytes
 * (map_rows).  With prompt_mask, a map row's keys are its own prompt 0's, and its token masks should all be 1 (no region):
 * maps of a regional sample are not defined.  map_batch = 0 is pb200_paella_features_tail, the same launches. */
int64_t pb200_paella_maps_workspace_bytes(const pb200_paella* m, int map_rows, int h, int w, int s_max);
int pb200_paella_features_maps(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_tail, int h, int w,
                               const void* cond_cache, int cache_slots, const int* kv_slot, int s_max, const float* attn_w, int n_w,
                               int w_ld, const int* w_len, const int* w_row, int w_batch, const uint8_t* wrap, const uint8_t* prompt_mask,
                               const int* mask_row, const int* region_slot, int max_regions, const int* tail_src, const int* map_row,
                               int map_batch, float* map_acc, int map_rows, int map_len, float* features, void* workspace,
                               int64_t workspace_bytes, void* stream);
/* Prompt-to-prompt injection: pb200_paella_features_maps where, in every AttnBlock and every head, base sample b < inj_batch
 * with a = inj_src[b] >= 0 (DEVICE int32 [inj_batch], -1: none; a < batch_total - n_tail, a != b) attends with sample a's
 * attention probabilities and its own values (pb200_attention_inject).  The caller keeps the conditioning lengths of b and a
 * equal, and neither is regional.  Rows that are not injected, the source rows among them, get the bits of the call without
 * injection.  inj_batch = 0 is pb200_paella_features_maps, the same launches. */
int pb200_paella_features_inject(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_tail, int h, int w,
                                 const void* cond_cache, int cache_slots, const int* kv_slot, int s_max, const float* attn_w, int n_w,
                                 int w_ld, const int* w_len, const int* w_row, int w_batch, const uint8_t* wrap,
                                 const uint8_t* prompt_mask, const int* mask_row, const int* region_slot, int max_regions,
                                 const int* tail_src, const int* map_row, int map_batch, float* map_acc, int map_rows, int map_len,
                                 const int* inj_src, int inj_batch, float* features, void* workspace, int64_t workspace_bytes,
                                 void* stream);
/* ------------------------------------------------------------------------------------------
 * LoRA adapters per sample on every AttnBlock: a sample with adapter (A, B, alpha) of rank r at scale s is computed as the
 * reference model with W' = W + s * (alpha / r) * B A on the adapter's targets, which are the projections of
 *   Attention2D / nn.MultiheadAttention in_proj (q, k, v packed) and out_proj   ref/src/modules.py:12-19
 *   AttnBlock.kv_mapper[1]                                                       ref/src/modules.py:76-79
 * Each delta is added after the layer's own GEMM by a segmented shrink (U = x A^T) + expand (y += s (alpha/r) U B^T) kernel.
 * ------------------------------------------------------------------------------------------ */
#define PB200_LORA_MAX_ADAPTERS 32        /* distinct adapters in one call */
#define PB200_LORA_MAX_ATTN_BLOCKS 128
#define PB200_LORA_WORKSPACE_PER_ROW 256  /* bytes of scratch per row: the shrink's fp32 U, up to 64 ranks */
enum { PB200_LORA_IN_PROJ = 1, PB200_LORA_OUT_PROJ = 2, PB200_LORA_KV_MAPPER = 4 };   /* target bits */

/* One adapter operand of the kernel-level entry point:
 *   a    fp16 [rank_pad][k] (rows >= r zero), b fp16 [n][rank_pad] (columns >= r zero), both 16-byte aligned;
 *   aux  fp32 [rank_pad + 1]: the row sums of the fp16 rows of a (read in folded-LayerNorm mode), then alpha / r;
 *   rank_pad  r rounded up to a multiple of 8 (8..64), 0 = absent. */
typedef struct pb200_lora_operand {
    const void* a;
    const void* b;
    const float* aux;
    int rank_pad;
} pb200_lora_operand;

/* For rows i < m with id = row_adapter[i / rows_per_entry] >= 0 (< n_ops) and s = row_scale[i / rows_per_entry] != 0 (DEVICE int32 /
 * fp32 tables):  u = x[i] a_id^T, or with ln_stat (DEVICE int64 [m][2], the PB200_EPI_F16_LN statistics over k columns of the
 * shifted fp16 rows x) u_j = rstd_i (x[i] a_id[j]^T - mean'_i aux[j]);  then y[o] += s * aux[rank_pad] * u b_id^T with
 * o = (i / remap_in) * remap_out + i % remap_in (remap_in = 0: o = i).  y: fp16 (y_f32 = 0, rounded once) or fp32, ldy elements
 * per row.  Rows with id -1 or scale 0 are neither read nor written.  Each row's result depends on its own row, adapter and scale
 * only (no split-K, no atomics, one summation order).  k % 8 == 0, ldx % 8 == 0, n and ldy even.  ops: HOST array of n_ops <= 32
 * operands.  workspace: m * PB200_LORA_WORKSPACE_PER_ROW bytes. */
int pb200_lora_shrink_expand(const void* x, int64_t ldx, int64_t m, int k, int n, int rows_per_entry, const int* row_adapter,
                             const float* row_scale, const pb200_lora_operand* ops, int n_ops, const int64_t* ln_stat, void* y,
                             int64_t ldy, int y_f32, int remap_in, int remap_out, void* workspace, int64_t workspace_bytes,
                             void* stream);

/* A packed adapter of a model (paella_b200/lora.py builds it).  blob: DEVICE, 256-byte aligned; rank 1..64; targets[i]: the target
 * bits AttnBlock i (plan order, i < n_attn) carries.  Blob layout, with rp = rank rounded up to a multiple of 8: for each AttnBlock in
 * plan order, for each target it carries in the order in_proj, out_proj, kv_mapper, three parts, each starting on a 256-byte boundary:
 *   A    fp16 [rp][in]     lora_A rows, rows >= rank zero
 *   B    fp16 [out][rp]    lora_B rows, columns >= rank zero
 *   aux  fp32 [rp + 1]     row sums of the fp16 A rows, then alpha / rank
 * with (in, out) = (c, 3c) for in_proj, (c, c) for out_proj and (c_cond, c) for kv_mapper, c the block's width. */
typedef struct pb200_lora_adapter {
    const void* blob;
    int rank;
    unsigned char targets[PB200_LORA_MAX_ATTN_BLOCKS];
} pb200_lora_adapter;

/* pb200_paella_prepare_cond with adapters: slot batch_offset + b is projected under adapter row_adapter[b] (DEVICE int32 [batch],
 * -1: none, else an index into the HOST array adapters[n_adapters]) at scale row_scale[b] (DEVICE fp32 [batch]): kv_mapper[1] and
 * the K/V rows of in_proj get the adapter's deltas.  n_adapters = 0 is pb200_paella_prepare_cond, the same launches. */
int pb200_paella_prepare_cond_lora(pb200_paella* m, const pb200_cond* cond, int batch, int batch_offset, int batch_total, int s_max,
                                   void* cond_cache, void* workspace, int64_t workspace_bytes, const pb200_lora_adapter* adapters,
                                   int n_adapters, const int* row_adapter, const float* row_scale, void* stream);
/* pb200_paella_features_inject with adapters: base sample b (< batch_total - n_tail) runs every AttnBlock's in_proj and out_proj
 * under adapter row_adapter[b] (DEVICE int32 [batch_total - n_tail], -1: none) at scale row_scale[b] (DEVICE fp32), and so does
 * each tail row, under its source sample's entry (the unconditional and guidance-prompt term rows of that sample).  Nothing runs
 * before the first AttnBlock, so the shared prefix is unchanged.  Rows without an adapter get the bits of the call without
 * adapters.  n_adapters = 0 is pb200_paella_features_inject, the same launches. */
int pb200_paella_features_lora(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_tail, int h, int w,
                               const void* cond_cache, int cache_slots, const int* kv_slot, int s_max, const float* attn_w, int n_w,
                               int w_ld, const int* w_len, const int* w_row, int w_batch, const uint8_t* wrap,
                               const uint8_t* prompt_mask, const int* mask_row, const int* region_slot, int max_regions,
                               const int* tail_src, const int* map_row, int map_batch, float* map_acc, int map_rows, int map_len,
                               const int* inj_src, int inj_batch, const pb200_lora_adapter* adapters, int n_adapters,
                               const int* row_adapter, const float* row_scale, float* features, void* workspace,
                               int64_t workspace_bytes, void* stream);
/* pb200_paella_features_lora with perturbed-attention guidance: row b < pag_batch (of all batch_total rows, tail rows included)
 * runs AttnBlock i (plan order, at most 64 AttnBlocks) as pb200_attention_perturb when bit i of pag_mask[b] is set (DEVICE uint64
 * [pag_batch]); every other block and every other part of its forward is the row's plain forward.  A perturbed row is not
 * regional, injected or a source.  Rows whose mask is 0 get the bits of the call without it.  pag_batch = 0 is
 * pb200_paella_features_lora, the same launches. */
int pb200_paella_features_pag(pb200_paella* m, const int64_t* tokens, const float* r, int batch_total, int n_tail, int h, int w,
                              const void* cond_cache, int cache_slots, const int* kv_slot, int s_max, const float* attn_w, int n_w,
                              int w_ld, const int* w_len, const int* w_row, int w_batch, const uint8_t* wrap,
                              const uint8_t* prompt_mask, const int* mask_row, const int* region_slot, int max_regions,
                              const int* tail_src, const int* map_row, int map_batch, float* map_acc, int map_rows, int map_len,
                              const int* inj_src, int inj_batch, const pb200_lora_adapter* adapters, int n_adapters,
                              const int* row_adapter, const float* row_scale, const uint64_t* pag_mask, int pag_batch,
                              float* features, void* workspace, int64_t workspace_bytes, void* stream);

/* maps fp32 [rows][s][h][w] from rows consecutive accumulator rows of pb200_paella_features_maps accumulated over n_steps
 * forwards: maps[row][j][y][x] = (1 / (n_steps * n_attn)) * sum over levels l, ascending, of
 * map_acc[row][j][off_l + (y / (patch << l)) * gw_l + x / (patch << l)] (nearest-neighbour upsampling); s <= map_len. */
int pb200_paella_attention_maps_finalize(pb200_paella* m, const float* map_acc, int rows, int map_len, int h, int w, int s, int n_steps,
                                         float* maps, void* stream);

/* Guidance prompts: the K-way guided mix, in place on fp32 features [samples][hw][c_out] (pb200_paella_features_tail's output).
 * Composed sample y reads rows[y * ld .. + ld) (DEVICE int32 sample indices: its conditional row c, its unconditional row u,
 * then its term rows t_1 .. t_J, -1 after its last term) and coef[y * ld .. + ld) (DEVICE fp32 a_c, a_u, a_1 .. a_J), and
 * writes t = fmaf(f_c, a_c, f_u * a_u), then t = fmaf(f_j, a_j, t) for each term in order, over row c.  With coefficients that
 * sum to 1 this is the mix of the logits (the out_mapper is linear after its LayerNorm); a sampler then takes row c with the
 * params (1, 0, 1/T).  2 <= ld <= 2 + PB200_MAX_GUIDANCE_PROMPTS; no two composed samples share a row c. */
#define PB200_MAX_GUIDANCE_PROMPTS 7
int pb200_paella_guidance_mix(pb200_paella* m, float* features, int hw, const int* rows, const float* coef, int n_composed, int ld,
                              void* stream);

/* out_mapper on features -> logits fp32 NCHW [B, num_labels, H*W]   (ref/src/modules.py:184-187,274) */
int pb200_paella_logits(pb200_paella* m, const float* features, int batch, int hw, float* logits_nchw,
                        void* workspace, int64_t workspace_bytes, void* stream);

/* Fused out_mapper + CFG + temperature + multinomial (ref/src/utils.py:44-50): logits never reach HBM.
 *   features: fp32 [(2B or B)*HW, c_out]: conditional rows first, then unconditional rows (if cfg_on).
 *   tokens_out int64 [B*HW].  Gumbel-max in the log domain on torch's Philox stream:
 *   argmax_k( l_k/T - log q_k ), q_k the same Exp(1) draw torch.multinomial would use. */
int pb200_paella_sample_tokens(pb200_paella* m, const float* features, int batch, int hw, int cfg_on, double cfg,
                               double temperature, uint64_t seed, uint64_t offset, int64_t* tokens_out,
                               void* workspace, int64_t workspace_bytes, void* stream);

/* pb200_paella_sample_tokens with one random stream per sample, in ONE launch over the batch (a list of per-sample
 * torch.Generators).  seed_offset: DEVICE uint64 [batch][2] = (seed, philox offset) of sample b's generator before the
 * draw; offsets are multiples of 4.  Sample b's rows draw exactly what pb200_paella_sample_tokens(batch = 1) draws on
 * (seed, offset) = seed_offset[b], through the same kernel family and MMA shape, and each generator is to be advanced by
 * pb200_philox_offset_increment(hw * num_labels).  hw * num_labels <= 2^29 (torch would split a larger draw).
 * pb200_paella_workspace_bytes(batch, ...) sizes the workspace. */
int pb200_paella_sample_tokens_per_sample(pb200_paella* m, const float* features, int batch, int hw, int cfg_on, double cfg,
                                          double temperature, const uint64_t* seed_offset, int64_t* tokens_out,
                                          void* workspace, int64_t workspace_bytes, void* stream);

/* pb200_paella_sample_tokens with per-sample guidance scale and temperature, in ONE launch over the batch.  params: DEVICE
 * float [batch][3] of per-sample (cfg, 1 - cfg, 1/T), as for pb200_resample_logits_params: row r of the CFG pre-mix uses
 * sample r / hw's (cfg, 1 - cfg) and its draw sample r / hw's 1/T.  seed_offset == NULL: one random stream (seed, offset)
 * over the batch, drawn exactly as pb200_paella_sample_tokens draws it; otherwise the per-sample (seed, offset) table of
 * pb200_paella_sample_tokens_per_sample (seed and offset are then ignored).  Either way sample b's tokens are those of the
 * scalar entry point on sample b's parameters. */
int pb200_paella_sample_tokens_params(pb200_paella* m, const float* features, int batch, int hw, int cfg_on, const float* params,
                                      uint64_t seed, uint64_t offset, const uint64_t* seed_offset, int64_t* tokens_out,
                                      void* workspace, int64_t workspace_bytes, void* stream);
/* pb200_paella_sample_tokens_params for the features of pb200_paella_features_pairs, per-sample streams only: features
 * fp32 [(batch + n_pairs)*HW, c_out]; samples b < n_pairs are guided (CFG mix with their rows at (batch + b)*HW), the others
 * draw on their conditional rows alone.  n_pairs in {0, batch} computes what pb200_paella_sample_tokens_params with
 * cfg_on = (n_pairs > 0) computes. */
int pb200_paella_sample_tokens_pairs(pb200_paella* m, const float* features, int batch, int n_pairs, int hw, const float* params,
                                     const uint64_t* seed_offset, int64_t* tokens_out, void* workspace, int64_t workspace_bytes,
                                     void* stream);
/* pb200_paella_sample_tokens_pairs for a batch in which some samples do not draw this step (they are sampled in another
 * mode, pb200_paella_resample_samples).  skip: int32 [batch]; a sample with skip[b] != 0 takes no part in the launch: its
 * rows of tokens_out are left as they are and its seed_offset entry is not read (its generator is not to be advanced).
 * Every other sample's tokens are those of pb200_paella_sample_tokens_pairs, which is this call with skip = NULL. */
int pb200_paella_sample_tokens_pairs_skip(pb200_paella* m, const float* features, int batch, int n_pairs, int hw, const float* params,
                                          const uint64_t* seed_offset, const int* skip, int64_t* tokens_out, void* workspace,
                                          int64_t workspace_bytes, void* stream);

/* Top-k / top-p truncated draws: pb200_paella_sample_tokens_params and pb200_paella_sample_tokens_pairs_skip with a per-sample
 * truncation table, top_k DEVICE int32 [batch] and top_p DEVICE float [batch] (both or neither; NULL is exactly the call
 * without the table, which is what the two functions above are).  For a token of sample b, with s_j = l_j * (1/T) the fp32
 * product of its guided logit and 1/T:
 *   top_k[b] = k >= 1: the kept set is {j : s_j >= tau_k}, tau_k the k-th largest s_j counting equal values separately (all
 *     ties at the boundary are kept); k >= num_labels keeps every label, still through the truncation kernels;
 *   top_p[b] = p in (0, 1): with w_j = exp(s_j - m) over the top-k kept set (m the row maximum), the kept set is
 *     {j : s_j >= tau_p}, tau_p the largest kept s_j with sum_{s_i >= tau_p} w_i >= p * sum w_i (boundary ties kept);
 *   the draw is unchanged: token = argmax over the kept j of (s_j - log q_j), the same Exp(1) variates at the same Philox
 *     elements as the untruncated call, so excluded labels still consume theirs and a generator advances as without truncation.
 * 0 and 1.0 are off; the tables are read on the device, so k < 0 and p outside (0, 1] are not diagnosed here (they are off).
 * Numerics: w_j is fp32 expf (<= 2 ulp) of the fp32 difference, summed as fixed-point floor(2^32 w_j) in 64-bit integers
 * (order-independent), and the mass test is evaluated in fp64 on those sums.  Truncation applies to the multinomial draw only. */
int pb200_paella_sample_tokens_params_trunc(pb200_paella* m, const float* features, int batch, int hw, int cfg_on,
                                            const float* params, uint64_t seed, uint64_t offset, const uint64_t* seed_offset,
                                            const int* top_k, const float* top_p, int64_t* tokens_out, void* workspace,
                                            int64_t workspace_bytes, void* stream);
int pb200_paella_sample_tokens_pairs_trunc(pb200_paella* m, const float* features, int batch, int n_pairs, int hw, const float* params,
                                           const uint64_t* seed_offset, const int* skip, const int* top_k, const float* top_p,
                                           int64_t* tokens_out, void* workspace, int64_t workspace_bytes, void* stream);

/* The notebook's non-multinomial sampling modes (paella_inference.ipynb cell 3) for a list of samples of the features of
 * pb200_paella_features_pairs, so that samples in different modes share one forward.  For each listed sample s the call
 * computes what pb200_paella_logits followed by pb200_resample_logits_params (mode = 1, argmax) or
 * pb200_resample_quant_params (mode = 2, quant: softmax @ codebook, then the nearest code) computes for that sample on its
 * own, and writes its tokens to rows [s*hw, (s+1)*hw) of tokens_out.  Neither mode draws a random number.
 *   features  fp32 [(batch + n_pairs)*hw, c_out]: sample s's rows at s*hw, a guided sample's unconditional rows at
 *             (batch + s)*hw;
 *   samples   int32 [n]: distinct sample indices; samples[0, n_guided) are guided (each < n_pairs) and are mixed with
 *             their unconditional logits, the others are not;
 *   params    fp32 [batch][3] of per-sample (cfg, 1 - cfg, 1/T), as for pb200_resample_logits_params;
 *   codebook  fp32 [num_labels][c_latent] for mode 2 (c_latent 1..8), ignored for mode 1.
 * The samples go through the out_mapper GEMM at most `chunk` guided (or 2*chunk unguided) at a time, so the logits scratch
 * is bounded by pb200_paella_resample_workspace_bytes(chunk, hw) = 2*chunk*hw*(2*c_out + 4*num_labels) bytes (rounded). */
int64_t pb200_paella_resample_workspace_bytes(const pb200_paella* m, int chunk, int hw);
int pb200_paella_resample_samples(pb200_paella* m, const float* features, int batch, int n_pairs, int hw, const int* samples, int n,
                                  int n_guided, const float* params, int mode, const float* codebook, int c_latent, int chunk,
                                  int64_t* tokens_out, void* workspace, int64_t workspace_bytes, void* stream);

/* Token scoring: per-token log-likelihood statistics of given codes under the denoiser, from one fused out_mapper +
 * log-softmax kernel; the logits never reach HBM.  Replaces ref/utils/modules.py:268-280 (the out_mapper of Paella.forward)
 * followed by src/train.py:36,64,71 (nn.CrossEntropyLoss(label_smoothing, reduction='none')(pred, latents) and
 * pred.argmax(1) == latents).
 *   features  fp32 [(batch + n_pairs)*hw, c_out] in pb200_paella_features_pairs layout: the first n_pairs samples are mixed
 *             with their unconditional rows at (batch + s)*hw using params' (cfg, 1 - cfg) (the A operand
 *             pb200_paella_sample_tokens_pairs draws from at T = 1), the others are taken as they are;
 *   params    fp32 [batch][3] of per-sample (cfg, 1 - cfg, 1/T), only the first two columns read; NULL when n_pairs = 0;
 *   targets   int64 [batch*hw] codes.
 * Per row, with l the logits and y the target: nll_out = logsumexp(l) - l_y, smooth_out = logsumexp(l) - mean_j l_j (fp32
 * [batch*hw] each; the label-smoothed loss is (1 - eps) nll + eps smooth) and argmax_out = the lowest j with l_j = max l
 * (int64 [batch*hw]).  A target outside [0, num_labels) gives a NaN nll in its row and nothing else: it is never used as an
 * index.  Each row's results depend only on its own features.  workspace: pb200_paella_token_scores_workspace_bytes(batch, hw)
 * bytes (the fp16 A operand). */
int64_t pb200_paella_token_scores_workspace_bytes(const pb200_paella* m, int batch, int hw);
int pb200_paella_token_scores(pb200_paella* m, const float* features, int batch, int n_pairs, int hw, const float* params,
                              const int64_t* targets, float* nll_out, float* smooth_out, int64_t* argmax_out, void* workspace,
                              int64_t workspace_bytes, void* stream);
/* The log-probability of each drawn token under the distribution the fused sampler drew it from, for confidence-guided
 * renoising: replaces the log_softmax(logits / T) the reference would materialise.  The rows and the n_pairs mix are
 * pb200_paella_token_scores's (the A operand pb200_paella_sample_tokens_pairs feeds the sampler; with n_pairs = 0 that of
 * pb200_paella_sample_tokens_params with cfg_on = 0), and params (fp32 [batch][3], required) also gives each sample's 1/T
 * (column 2).  logp_out fp32 [batch*hw] = s_y - logsumexp(s), s = l * (1/T) rounded once per logit, y = tokens[row]; at 1/T = 1
 * this is -nll of pb200_paella_token_scores bit for bit.  workspace: pb200_paella_token_scores_workspace_bytes(batch, hw). */
int pb200_paella_token_logprob(pb200_paella* m, const float* features, int batch, int n_pairs, int hw, const float* params,
                               const int64_t* tokens, float* logp_out, void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * VQGAN (ref/src/vqgan.py:45-107).
 * ------------------------------------------------------------------------------------------ */
typedef struct pb200_vqgan_config {   /* VQModel kwargs, ref/src/vqgan.py:46-47 */
    int levels, bottleneck_blocks, c_hidden, c_latent, codebook_size;
    float scale_factor;
} pb200_vqgan_config;

typedef struct pb200_vqgan pb200_vqgan;

int pb200_vqgan_create(const pb200_vqgan_config* cfg, pb200_vqgan** out);
void pb200_vqgan_destroy(pb200_vqgan* m);
int64_t pb200_vqgan_weight_bytes(const pb200_vqgan* m);
int pb200_vqgan_bind_weights(pb200_vqgan* m, void* weight_blob);
int pb200_vqgan_num_params(const pb200_vqgan* m);
const char* pb200_vqgan_param_name(const pb200_vqgan* m, int i);
int64_t pb200_vqgan_param_numel(const pb200_vqgan* m, int i);
int pb200_vqgan_load_param(pb200_vqgan* m, const char* name, const float* src, int64_t numel, void* stream);
int64_t pb200_vqgan_workspace_bytes(const pb200_vqgan* m, int batch, int img_h, int img_w);

/* VQModel.encode: img fp32 NCHW [B,3,H,W] -> latents fp32 NCHW [B,c_latent,H/4,W/4] (pre-quantisation,
 * NOT divided by scale_factor), quantised latents (same shape) and indices int64 [B,H/4,W/4]. */
int pb200_vqgan_encode(pb200_vqgan* m, const float* img, int batch, int img_h, int img_w, float* latents_nchw,
                       float* quantised_nchw, int64_t* indices, void* workspace, int64_t workspace_bytes,
                       void* stream);
/* VQModel.decode_indices (indices != NULL) or VQModel.decode on NCHW latents already multiplied by
 * scale_factor (latents_nchw != NULL) -> img fp32 NCHW [B,3,4h,4w]. */
int pb200_vqgan_decode(pb200_vqgan* m, const int64_t* indices, const float* latents_nchw, int batch, int h, int w,
                       float* img, void* workspace, int64_t workspace_bytes, void* stream);

/* One codec ResBlock on its own (ref/src/vqgan.py:36-42) -- what `vqgan.ResBlock.forward` runs outside a VQModel; inside
 * one, encode/decode run the same kernels from the plan.  x_nhwc fp32 [B,h,w,c] is updated in place; dw_w9 = the depthwise
 * kernel as [9][c] fp32 (tap-major), w1 [4c,c] / w2 [c,4c] fp16 row-major, gammas_host = the 6 scalars (HOST memory). */
int64_t pb200_vqgan_resblock_workspace_bytes(int batch, int h, int w, int c);
int pb200_vqgan_resblock(float* x_nhwc, int batch, int h, int w, int c, const float* dw_w9, const float* dw_bias,
                         const void* w1_f16, const float* b1, const void* w2_f16, const float* b2, const float* gammas_host,
                         void* workspace, int64_t workspace_bytes, void* stream);

/* Output forms of the decoder's last kernel (out_block: 1x1 conv + PixelShuffle, ref/src/vqgan.py:86-89), fused with what
 * the reference's callers do next (ref/src_distributed/train.py:168-171 `decode_indices(x).clamp(0, 1)`, then
 * torchvision.utils.save_image's `mul(255).add_(0.5).clamp_(0, 255).to(uint8)` on an HWC view):
 *   PB200_IMG_F32_NCHW          fp32 [B,3,4h,4w], unclamped               == pb200_vqgan_decode
 *   PB200_IMG_F32_NCHW_CLAMP01  fp32 [B,3,4h,4w], clamp(0,1)
 *   PB200_IMG_U8_NHWC           uint8 [B,4h,4w,3] = trunc(clamp(v,0,1)*255 + 0.5)   */
enum { PB200_IMG_F32_NCHW = 0, PB200_IMG_F32_NCHW_CLAMP01 = 1, PB200_IMG_U8_NHWC = 2 };
int pb200_vqgan_decode_ex(pb200_vqgan* m, const int64_t* indices, const float* latents_nchw, int batch, int h, int w,
                          void* img, int img_mode, void* workspace, int64_t workspace_bytes, void* stream);
/* pb200_vqgan_decode_ex with seamless tiling: wrap = DEVICE uint8 [batch] (bit 0 wraps x, bit 1 wraps y).  On a wrapped axis
 * the ResBlocks' ReplicationPad2d becomes circular padding and ConvTranspose2d(k4, s2, p1) reads its input indices modulo the
 * grid, so decode(roll(tokens, (a, b))) == roll(decode(tokens), (4a, 4b)).  wrap = NULL is pb200_vqgan_decode_ex; a byte-0
 * sample gives its bits. */
int pb200_vqgan_decode_tiled(pb200_vqgan* m, const int64_t* indices, const float* latents_nchw, int batch, int h, int w,
                             void* img, int img_mode, const uint8_t* wrap, void* workspace, int64_t workspace_bytes,
                             void* stream);

/* Re-read the host-mirrored scalars (the six ResBlock gammas, kernel arguments) from the bound weight blob.  Needed when
 * the blob was filled by anything other than pb200_vqgan_load_param on this handle (NCCL broadcast, a packed file,
 * cudaMemcpy).  bind_weights marks them stale and encode/decode refresh lazily (one stream synchronisation), so calling
 * this is only required when the blob CONTENT changes under an already-bound pointer.  Synchronises `stream`. */
int pb200_vqgan_sync_params(pb200_vqgan* m, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PAELLA_B200_H */
