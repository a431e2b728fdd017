// Random streams + the resample step of the sampling loop, reproducing PyTorch's CUDA
// generator (Philox4x32-10) element for element.
//   torch.randint        ref/src/utils.py:37
//   torch.multinomial    ref/src/utils.py:49-50   (q = exponential_(1); argmax(p / q))
//   CFG/temp/softmax     ref/src/utils.py:45-47
//   Paella.add_noise     ref/src/modules.py:277-283  (and its explicit-mask form, the region sampling of utils._sample_core)
// PyTorch-side arithmetic: ATen/native/cuda/DistributionTemplates.h, ATen/core/TransformationHelper.h.
#include "common.cuh"
#include "ops.cuh"
#include "paella_b200.h"

#include <float.h>

namespace pb {

TorchPhilox make_torch_philox(uint64_t seed, uint64_t offset, long numel) {
    const long block = 256;
    long grid = (numel + block - 1) / block;
    const long cap = (long)sm_count() * (max_threads_per_sm() / block);
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    TorchPhilox s;
    s.seed = seed;
    s.offset4 = offset / 4;
    s.stride = (uint32_t)(block * grid);
    return s;
}

static int64_t offset_increment(int64_t numel) {
    if (numel <= 0) return 0;
    TorchPhilox s = make_torch_philox(0, 0, numel);
    return ((numel - 1) / ((int64_t)s.stride * 4) + 1) * 4;
}

// ------------------------------------------------------------------ randint / rand
__global__ void randint_kernel(int64_t* __restrict__ out, int64_t numel, uint32_t range, TorchPhilox s) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= numel) return;
    out[e] = (int64_t)(torch_philox_u32(s, (uint64_t)e) % range);
}

__global__ void rand_kernel(float* __restrict__ out, int64_t numel, TorchPhilox s) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= numel) return;
    const float u = u32_to_uniform(torch_philox_u32(s, (uint64_t)e));
    out[e] = (u == 1.0f) ? 0.0f : u;     // uniform_kernel: value == to ? from : value
}

// ------------------------------------------------------------------ add_noise
// src, region (both NULL, or both set; indexed like random_x): region sampling.  Where region[e] == 0 the output is src[e]
// and the mask is 0: torch.where(region, add_noise(x, t, mask=m & region, random_x), src), the draw unchanged.
__global__ void add_noise_kernel(const int64_t* __restrict__ x, const int64_t* __restrict__ random_x,
                                 const int64_t* __restrict__ src, const uint8_t* __restrict__ region,
                                 const float* __restrict__ t, int64_t batch, int64_t hw, uint32_t num_labels,
                                 TorchPhilox s_mask, TorchPhilox s_rx, int64_t* __restrict__ out,
                                 int64_t* __restrict__ mask_out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= batch * hw) return;
    float u = u32_to_uniform(torch_philox_u32(s_mask, (uint64_t)e));
    u = (u == 1.0f) ? 0.0f : u;
    const bool gen = region ? region[e] != 0 : true;
    const bool m = gen && u <= t[e / hw];
    const int64_t rx = random_x ? random_x[e] : (int64_t)(torch_philox_u32(s_rx, (uint64_t)e) % num_labels);
    out[e] = gen ? (m ? rx : x[e]) : src[e];
    if (mask_out) mask_out[e] = m ? 1 : 0;
}

// ------------------------------------------------------------------ one random stream per sample, one launch
// Sample b = blockIdx.y draws on its own generator: (seed, philox offset) = seed_off[2b], seed_off[2b + 1], with the stride of
// s (the launch policy of ONE sample's draw of hw elements), so element e of sample b is element e of the batch-1 launch on
// that generator.  slot (int32 [B] or NULL = identity) places sample b's row of random_x and of out at slot[b] * hw.
__device__ __forceinline__ TorchPhilox sample_stream(TorchPhilox s, const uint64_t* __restrict__ seed_off, int64_t b) {
    s.seed = seed_off[2 * b];
    s.offset4 = seed_off[2 * b + 1] >> 2;
    return s;
}

__global__ void randint_per_sample_kernel(int64_t* __restrict__ out, const int* __restrict__ slot, int64_t hw, uint32_t range,
                                          TorchPhilox s, const uint64_t* __restrict__ seed_off) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= hw) return;
    const int64_t b = blockIdx.y;
    const int64_t dst = slot ? slot[b] : b;
    out[dst * hw + e] = (int64_t)(torch_philox_u32(sample_stream(s, seed_off, b), (uint64_t)e) % range);
}

// x: int64 [B, hw] (by sample); t: fp32 [B], and a sample with t < 0 keeps x (u >= 0 never passes the mask test: the
// sampling engine's rows that do not renoise this step).  random_x == NULL: randint_like drawn at the offset after the mask
// draw, as pb200_add_noise does (rx_inc4 = that offset increment / 4).  src, region: as in add_noise_kernel, by slot.
__global__ void add_noise_per_sample_kernel(const int64_t* __restrict__ x, const int64_t* __restrict__ random_x,
                                            const int64_t* __restrict__ src, const uint8_t* __restrict__ region,
                                            const int* __restrict__ slot, const float* __restrict__ t, int64_t hw,
                                            uint32_t num_labels, TorchPhilox s, uint64_t rx_inc4,
                                            const uint64_t* __restrict__ seed_off, int64_t* __restrict__ out,
                                            int64_t* __restrict__ mask_out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= hw) return;
    const int64_t b = blockIdx.y;
    const int64_t dst = slot ? slot[b] : b;
    const TorchPhilox sm = sample_stream(s, seed_off, b);
    float u = u32_to_uniform(torch_philox_u32(sm, (uint64_t)e));
    u = (u == 1.0f) ? 0.0f : u;
    const bool gen = region ? region[dst * hw + e] != 0 : true;
    const bool m = gen && u <= t[b];
    int64_t rx;
    if (random_x) {
        rx = random_x[dst * hw + e];
    } else {
        TorchPhilox sr = sm;
        sr.offset4 += rx_inc4;
        rx = (int64_t)(torch_philox_u32(sr, (uint64_t)e) % num_labels);
    }
    out[dst * hw + e] = gen ? (m ? rx : x[b * hw + e]) : src[dst * hw + e];
    if (mask_out) mask_out[b * hw + e] = m ? 1 : 0;
}

// out[b] = pool[slot[b]] for rows of hw tokens: the sampling engine's batch of one step, in that step's row order
__global__ void gather_rows_kernel(const int64_t* __restrict__ pool, const int* __restrict__ slot, int64_t hw,
                                   int64_t* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= hw) return;
    const int64_t b = blockIdx.y;
    out[b * hw + e] = pool[(int64_t)slot[b] * hw + e];
}

// ------------------------------------------------------------------ multinomial(p, 1): argmax p/q, first index on ties
struct ArgBest {
    float v;
    int idx;
};
__device__ __forceinline__ ArgBest better(ArgBest a, ArgBest b) {
    // torch argmax: larger value wins, lower index on ties (inputs are NaN-free: torch asserts p valid)
    const bool take_b = (b.v > a.v) || (b.v == a.v && b.idx < a.idx);
    return take_b ? b : a;
}
__device__ __forceinline__ ArgBest warp_best(ArgBest a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ArgBest b;
        b.v = __shfl_xor_sync(0xffffffffu, a.v, o);
        b.idx = __shfl_xor_sync(0xffffffffu, a.idx, o);
        a = better(a, b);
    }
    return a;
}

__global__ void __launch_bounds__(256) multinomial_kernel(const float* __restrict__ p, int64_t rows, int k, TorchPhilox s,
                                                          int64_t* __restrict__ out) {
    const int64_t row = blockIdx.x;
    const float* pr = p + row * k;
    ArgBest best{-INFINITY, 0x7fffffff};
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        const uint64_t e = (uint64_t)row * (uint64_t)k + (uint64_t)j;
        const float q = torch_exponential1(u32_to_uniform(torch_philox_u32(s, e)));
        const float v = __fdiv_rn(pr[j], q);
        best = better(best, ArgBest{v, j});
    }
    __shared__ float sv[8];
    __shared__ int si[8];
    best = warp_best(best);
    if ((threadIdx.x & 31) == 0) {
        sv[threadIdx.x >> 5] = best.v;
        si[threadIdx.x >> 5] = best.idx;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        ArgBest b{-INFINITY, 0x7fffffff};
        if (threadIdx.x < (blockDim.x >> 5)) b = ArgBest{sv[threadIdx.x], si[threadIdx.x]};
        b = warp_best(b);
        if (threadIdx.x == 0) out[row] = b.idx;
    }
}

// ------------------------------------------------------------------ resample on reference-layout logits
// One CTA = 32 consecutive positions p of one sample (coalesced along HW) x all K, 8 warps stride K.
//   l  = lc*cfg + lu*(1-cfg)          (two rounded products and a rounded sum, like the three torch kernels)
//   l' = l * (1/T)                    (torch's div-by-CPU-scalar fast path multiplies by the reciprocal)
//   p  = exp(l' - max) / sum          (softmax dim=1)
//   tok = argmax_k p_k / q_k
// params (may be null): DEVICE [B][3] per-sample (cfg, 1 - cfg, 1/T), replacing the three scalars for sample b = blockIdx.y.
// map (may be null): DEVICE int32 [gridDim.y]; the logits of launch sample b = blockIdx.y are those of output sample map[b],
// whose params row and token row it uses -- a packed launch over some samples writes straight into the batch's rows.
template <int MODE>
__global__ void __launch_bounds__(256, 4) resample_logits_kernel(const float* __restrict__ lc, const float* __restrict__ lu,
                                                                 int k, int64_t hw, float cfg_arg, float one_minus_cfg_arg,
                                                                 float inv_t_arg, const float* __restrict__ params, TorchPhilox s,
                                                                 const int* __restrict__ map, int64_t* __restrict__ out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t b = blockIdx.y;
    const int64_t ob = map ? (int64_t)map[b] : b;       // output sample
    const float cfg = params ? params[3 * ob] : cfg_arg;
    const float one_minus_cfg = params ? params[3 * ob + 1] : one_minus_cfg_arg;
    const float inv_t = params ? params[3 * ob + 2] : inv_t_arg;
    const int64_t pos = (int64_t)blockIdx.x * 32 + lane;
    const bool valid = pos < hw;
    const float* c_ptr = lc + b * (int64_t)k * hw + (valid ? pos : 0);
    const float* u_ptr = lu ? lu + b * (int64_t)k * hw + (valid ? pos : 0) : nullptr;
    __shared__ float red[8][33];
    __shared__ int redi[8][33];

    auto mixed = [&](int j) -> float {
        float l = c_ptr[(int64_t)j * hw];
        if (u_ptr) l = __fadd_rn(__fmul_rn(l, cfg), __fmul_rn(u_ptr[(int64_t)j * hw], one_minus_cfg));
        return l;
    };

    if (MODE == 1) {   // argmax of the (guided) logits
        ArgBest best{-INFINITY, 0x7fffffff};
        for (int j = warp; j < k; j += 8) best = better(best, ArgBest{mixed(j), j});
        red[warp][lane] = best.v;
        redi[warp][lane] = best.idx;
        __syncthreads();
        if (warp == 0) {
            ArgBest bb{red[0][lane], redi[0][lane]};
            for (int w = 1; w < 8; ++w) bb = better(bb, ArgBest{red[w][lane], redi[w][lane]});
            if (valid) out[ob * hw + pos] = bb.idx;
        }
        return;
    }

    // pass 1: max
    float m = -INFINITY;
    for (int j = warp; j < k; j += 8) m = fmaxf(m, __fmul_rn(mixed(j), inv_t));
    red[warp][lane] = m;
    __syncthreads();
    m = red[0][lane];
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w][lane]);
    __syncthreads();
    // pass 2: sum of exp
    float sum = 0.f;
    for (int j = warp; j < k; j += 8) sum += expf(__fmul_rn(mixed(j), inv_t) - m);
    red[warp][lane] = sum;
    __syncthreads();
    sum = red[0][lane];
    for (int w = 1; w < 8; ++w) sum += red[w][lane];
    __syncthreads();
    // pass 3: argmax p/q
    ArgBest best{-INFINITY, 0x7fffffff};
    if (valid) {
        const uint64_t row = (uint64_t)(b * hw + pos);
        for (int j = warp; j < k; j += 8) {
            const float pj = __fdiv_rn(expf(__fmul_rn(mixed(j), inv_t) - m), sum);
            const float q = torch_exponential1(u32_to_uniform(torch_philox_u32(s, row * (uint64_t)k + (uint64_t)j)));
            best = better(best, ArgBest{__fdiv_rn(pj, q), j});
        }
    }
    red[warp][lane] = best.v;
    redi[warp][lane] = best.idx;
    __syncthreads();
    if (warp == 0 && valid) {
        ArgBest bb{red[0][lane], redi[0][lane]};
        for (int w = 1; w < 8; ++w) bb = better(bb, ArgBest{red[w][lane], redi[w][lane]});
        out[b * hw + pos] = bb.idx;
    }
}

// ------------------------------------------------------------------ `quant` sampling mode (notebook cell 3, ref/src_distributed/train.py:155-156)
//   e = softmax(l / T) @ codebook  [C values per token];  token = nearest code of e   (deterministic, no draw)
// Same CTA shape as resample_logits_kernel: 32 positions x 8 warps striding the labels.
template <int C>
__global__ void __launch_bounds__(256) resample_quant_kernel(const float* __restrict__ lc, const float* __restrict__ lu, int k,
                                                             int64_t hw, float cfg_arg, float one_minus_cfg_arg, float inv_t_arg,
                                                             const float* __restrict__ params, const float* __restrict__ codebook,
                                                             const int* __restrict__ map, int64_t* __restrict__ out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t b = blockIdx.y;
    const int64_t ob = map ? (int64_t)map[b] : b;       // output sample, as in resample_logits_kernel
    const float cfg = params ? params[3 * ob] : cfg_arg;                  // per-sample parameters as in resample_logits
    const float one_minus_cfg = params ? params[3 * ob + 1] : one_minus_cfg_arg;
    const float inv_t = params ? params[3 * ob + 2] : inv_t_arg;
    const int64_t pos = (int64_t)blockIdx.x * 32 + lane;
    const bool valid = pos < hw;
    const float* c_ptr = lc + b * (int64_t)k * hw + (valid ? pos : 0);
    const float* u_ptr = lu ? lu + b * (int64_t)k * hw + (valid ? pos : 0) : nullptr;
    __shared__ float red[8][33];
    __shared__ float redc[C][8][33];
    __shared__ int redi[8][33];
    auto mixed = [&](int j) -> float {
        float l = c_ptr[(int64_t)j * hw];
        if (u_ptr) l = __fadd_rn(__fmul_rn(l, cfg), __fmul_rn(u_ptr[(int64_t)j * hw], one_minus_cfg));
        return __fmul_rn(l, inv_t);
    };
    float m = -INFINITY;
    for (int j = warp; j < k; j += 8) m = fmaxf(m, mixed(j));
    red[warp][lane] = m;
    __syncthreads();
    m = red[0][lane];
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w][lane]);
    __syncthreads();
    float sum = 0.f, acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0.f;
    for (int j = warp; j < k; j += 8) {
        const float e = expf(mixed(j) - m);
        sum += e;
#pragma unroll
        for (int c = 0; c < C; ++c) acc[c] = fmaf(e, __ldg(codebook + (int64_t)j * C + c), acc[c]);
    }
    red[warp][lane] = sum;
#pragma unroll
    for (int c = 0; c < C; ++c) redc[c][warp][lane] = acc[c];
    __syncthreads();
    sum = 0.f;
    float x[C];
#pragma unroll
    for (int c = 0; c < C; ++c) x[c] = 0.f;
    for (int w = 0; w < 8; ++w) {
        sum += red[w][lane];
#pragma unroll
        for (int c = 0; c < C; ++c) x[c] += redc[c][w][lane];
    }
    float x2 = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) { x[c] = __fdiv_rn(x[c], sum); x2 = fmaf(x[c], x[c], x2); }
    // nearest code (same arithmetic as vq_nearest_kernel), codes strided over the 8 warps
    float best = INFINITY;
    int bi = 0x7fffffff;
    for (int j = warp; j < k; j += 8) {
        float c2 = 0.f, dot = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const float cv = __ldg(codebook + (int64_t)j * C + c);
            c2 = fmaf(cv, cv, c2);
            dot = fmaf(x[c], cv, dot);
        }
        const float d = fmaf(-2.0f, dot, __fadd_rn(c2, x2));
        if (d < best) { best = d; bi = j; }
    }
    __syncthreads();
    red[warp][lane] = best;
    redi[warp][lane] = bi;
    __syncthreads();
    if (warp == 0 && valid) {
        float bd = red[0][lane];
        int bj = redi[0][lane];
        for (int w = 1; w < 8; ++w)
            if (red[w][lane] < bd || (red[w][lane] == bd && redi[w][lane] < bj)) { bd = red[w][lane]; bj = redi[w][lane]; }
        out[ob * hw + pos] = bj;
    }
}

}  // namespace pb

using namespace pb;

extern "C" {

int64_t pb200_philox_offset_increment(int64_t numel) { return offset_increment(numel); }

int pb200_randint(int64_t* out, int64_t numel, int64_t num_labels, uint64_t seed, uint64_t offset, void* stream) {
    PB_CHECK(num_labels > 0 && num_labels < (1ll << 28), "randint: range %lld needs the 64-bit path (unsupported)",
             (long long)num_labels);
    PB_CHECK(offset % 4 == 0, "philox offset must be a multiple of 4");
    if (numel == 0) return 0;
    TorchPhilox s = make_torch_philox(seed, offset, numel);
    randint_kernel<<<ceil_div(numel, 256), 256, 0, (cudaStream_t)stream>>>(out, numel, (uint32_t)num_labels, s);
    PB_LAUNCH_CHECK();
    return 0;
}

int pb200_rand(float* out, int64_t numel, uint64_t seed, uint64_t offset, void* stream) {
    PB_CHECK(offset % 4 == 0, "philox offset must be a multiple of 4");
    if (numel == 0) return 0;
    TorchPhilox s = make_torch_philox(seed, offset, numel);
    rand_kernel<<<ceil_div(numel, 256), 256, 0, (cudaStream_t)stream>>>(out, numel, s);
    PB_LAUNCH_CHECK();
    return 0;
}

int pb200_multinomial(const float* p, int64_t rows, int64_t k, uint64_t seed, uint64_t offset, int64_t* out,
                      void* stream) {
    PB_CHECK(offset % 4 == 0, "philox offset must be a multiple of 4");
    PB_CHECK(k > 0 && k < (1ll << 30), "multinomial: bad category count");
    PB_CHECK(rows * k < (1ll << 31), "multinomial: rows*k >= 2^31 would split the torch kernel (unsupported)");
    if (rows == 0) return 0;
    TorchPhilox s = make_torch_philox(seed, offset, rows * k);
    multinomial_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(p, rows, (int)k, s, out);
    PB_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"

namespace pb {
// python scalars: `logits * cfg` and `(1 - cfg)` are doubles cast to the fp32 op-math type; `temperatures[i]` is an fp32
// 0-dim CPU tensor and torch multiplies by its fp32 reciprocal.  These are the fp32 constants a per-sample table holds too.
static int resample_logits(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw, double cfg,
                           double temperature, const float* params, int mode, uint64_t seed, uint64_t offset, int64_t* out,
                           cudaStream_t st, const int* map = nullptr) {
    PB_CHECK(offset % 4 == 0, "philox offset must be a multiple of 4");
    PB_CHECK(map == nullptr || mode == 1, "resample: an output map is for argmax only");
    PB_CHECK(mode == 0 || mode == 1, "resample: mode must be 0 (multinomial) or 1 (argmax)");
    PB_CHECK(batch * hw * k < (1ll << 31), "resample: B*HW*K >= 2^31 would split the torch kernel (unsupported)");
    if (batch == 0 || hw == 0) return 0;
    TorchPhilox s = make_torch_philox(seed, offset, batch * hw * k);
    const float cfg_f = (float)cfg;
    const float one_minus = (float)(1.0 - cfg);
    const float inv_t = 1.0f / (float)temperature;
    dim3 grid(ceil_div(hw, 32), (unsigned)batch);
    if (mode == 0)
        resample_logits_kernel<0><<<grid, 256, 0, st>>>(logits_c, logits_u, (int)k, hw, cfg_f, one_minus, inv_t, params, s, nullptr, out);
    else
        resample_logits_kernel<1><<<grid, 256, 0, st>>>(logits_c, logits_u, (int)k, hw, cfg_f, one_minus, inv_t, params, s, map, out);
    PB_LAUNCH_CHECK();
    return 0;
}

static int resample_quant(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw, double cfg,
                          double temperature, const float* params, const float* codebook, int c_latent, int64_t* out,
                          cudaStream_t st, const int* map = nullptr) {
    PB_CHECK(c_latent >= 1 && c_latent <= 8, "resample_quant: c_latent %d unsupported (1..8)", c_latent);
    if (batch == 0 || hw == 0) return 0;
    const float cfg_f = (float)cfg, one_minus = (float)(1.0 - cfg), inv_t = 1.0f / (float)temperature;
    dim3 grid(ceil_div(hw, 32), (unsigned)batch);
    switch (c_latent) {
#define PB_RQ_CASE(C) \
    case C: resample_quant_kernel<C><<<grid, 256, 0, st>>>(logits_c, logits_u, (int)k, hw, cfg_f, one_minus, inv_t, params, codebook, map, out); break;
        PB_RQ_CASE(1) PB_RQ_CASE(2) PB_RQ_CASE(3) PB_RQ_CASE(4) PB_RQ_CASE(5) PB_RQ_CASE(6) PB_RQ_CASE(7) PB_RQ_CASE(8)
#undef PB_RQ_CASE
    }
    PB_LAUNCH_CHECK();
    return 0;
}

int launch_resample_mapped(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw, const float* params,
                           const int* map, int mode, const float* codebook, int c_latent, int64_t* out, cudaStream_t st) {
    PB_CHECK(params != nullptr && map != nullptr, "resample_mapped: params and map are required");
    PB_CHECK(batch <= 65535, "resample_mapped: %lld samples in one launch (grid.y)", (long long)batch);
    if (mode == 1) return resample_logits(logits_c, logits_u, batch, k, hw, 0.0, 1.0, params, 1, 0, 0, out, st, map);
    PB_CHECK(mode == 2, "resample_mapped: mode %d (1 = argmax, 2 = quant)", mode);
    return resample_quant(logits_c, logits_u, batch, k, hw, 0.0, 1.0, params, codebook, c_latent, out, st, map);
}
}  // namespace pb

extern "C" {

int pb200_resample_logits(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw,
                          double cfg, double temperature, int mode, uint64_t seed, uint64_t offset, int64_t* out,
                          void* stream) {
    return resample_logits(logits_c, logits_u, batch, k, hw, cfg, temperature, nullptr, mode, seed, offset, out,
                           (cudaStream_t)stream);
}

int pb200_resample_logits_params(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw,
                                 const float* params, int mode, uint64_t seed, uint64_t offset, int64_t* out, void* stream) {
    PB_CHECK(params != nullptr, "resample_logits_params: params is NULL");
    return resample_logits(logits_c, logits_u, batch, k, hw, 0.0, 1.0, params, mode, seed, offset, out, (cudaStream_t)stream);
}

int pb200_resample_quant(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw, double cfg,
                         double temperature, const float* codebook, int c_latent, int64_t* out, void* stream) {
    return resample_quant(logits_c, logits_u, batch, k, hw, cfg, temperature, nullptr, codebook, c_latent, out,
                          (cudaStream_t)stream);
}

int pb200_resample_quant_params(const float* logits_c, const float* logits_u, int64_t batch, int64_t k, int64_t hw,
                                const float* params, const float* codebook, int c_latent, int64_t* out, void* stream) {
    PB_CHECK(params != nullptr, "resample_quant_params: params is NULL");
    return resample_quant(logits_c, logits_u, batch, k, hw, 0.0, 1.0, params, codebook, c_latent, out, (cudaStream_t)stream);
}

int pb200_add_noise_region(const int64_t* x, const int64_t* random_x, const int64_t* src, const uint8_t* region, const float* t,
                           int64_t batch, int64_t hw, int64_t num_labels, uint64_t seed, uint64_t offset, int64_t* out,
                           int64_t* mask_out, void* stream) {
    PB_CHECK(offset % 4 == 0, "philox offset must be a multiple of 4");
    PB_CHECK(num_labels > 0 && num_labels < (1ll << 28), "add_noise: bad num_labels");
    PB_CHECK((src == nullptr) == (region == nullptr), "add_noise_region: src and region must both be set or both be NULL");
    const int64_t n = batch * hw;
    if (n == 0) return 0;
    TorchPhilox s_mask = make_torch_philox(seed, offset, n);
    TorchPhilox s_rx = make_torch_philox(seed, offset + offset_increment(n), n);
    add_noise_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(x, random_x, src, region, t, batch, hw,
                                                                         (uint32_t)num_labels, s_mask, s_rx, out, mask_out);
    PB_LAUNCH_CHECK();
    return 0;
}

int pb200_add_noise(const int64_t* x, const int64_t* random_x, const float* t, int64_t batch, int64_t hw,
                    int64_t num_labels, uint64_t seed, uint64_t offset, int64_t* out, int64_t* mask_out,
                    void* stream) {
    return pb200_add_noise_region(x, random_x, nullptr, nullptr, t, batch, hw, num_labels, seed, offset, out, mask_out, stream);
}

static int check_per_sample(int64_t batch, int64_t hw, const uint64_t* seed_offset, const char* what) {
    PB_CHECK(seed_offset != nullptr, "%s: per-sample (seed, offset) table is NULL", what);
    PB_CHECK(batch >= 0 && batch <= 65535, "%s: batch %lld out of range (<= 65535)", what, (long long)batch);
    PB_CHECK(hw >= 0 && hw <= (1ll << 29), "%s: a per-sample draw of %lld elements (> 2^29) would split the torch kernel", what,
             (long long)hw);
    return 0;
}

int pb200_randint_per_sample(int64_t* out, const int* slot, int64_t batch, int64_t hw, int64_t num_labels,
                             const uint64_t* seed_offset, void* stream) {
    PB_TRY(check_per_sample(batch, hw, seed_offset, "randint_per_sample"));
    PB_CHECK(num_labels > 0 && num_labels < (1ll << 28), "randint_per_sample: range %lld needs the 64-bit path (unsupported)",
             (long long)num_labels);
    if (batch == 0 || hw == 0) return 0;
    const TorchPhilox s = make_torch_philox(0, 0, hw);
    randint_per_sample_kernel<<<dim3(ceil_div(hw, 256), (unsigned)batch), 256, 0, (cudaStream_t)stream>>>(
        out, slot, hw, (uint32_t)num_labels, s, seed_offset);
    PB_LAUNCH_CHECK();
    return 0;
}

int pb200_add_noise_region_per_sample(const int64_t* x, const int64_t* random_x, const int64_t* src, const uint8_t* region,
                                      const int* slot, const float* t, int64_t batch, int64_t hw, int64_t num_labels,
                                      const uint64_t* seed_offset, int64_t* out, int64_t* mask_out, void* stream) {
    PB_TRY(check_per_sample(batch, hw, seed_offset, "add_noise_per_sample"));
    PB_CHECK(num_labels > 0 && num_labels < (1ll << 28), "add_noise_per_sample: bad num_labels");
    PB_CHECK((src == nullptr) == (region == nullptr), "add_noise_region_per_sample: src and region must both be set or both be NULL");
    if (batch == 0 || hw == 0) return 0;
    const TorchPhilox s = make_torch_philox(0, 0, hw);
    add_noise_per_sample_kernel<<<dim3(ceil_div(hw, 256), (unsigned)batch), 256, 0, (cudaStream_t)stream>>>(
        x, random_x, src, region, slot, t, hw, (uint32_t)num_labels, s, (uint64_t)offset_increment(hw) / 4, seed_offset, out,
        mask_out);
    PB_LAUNCH_CHECK();
    return 0;
}

int pb200_add_noise_per_sample(const int64_t* x, const int64_t* random_x, const int* slot, const float* t, int64_t batch,
                               int64_t hw, int64_t num_labels, const uint64_t* seed_offset, int64_t* out, int64_t* mask_out,
                               void* stream) {
    return pb200_add_noise_region_per_sample(x, random_x, nullptr, nullptr, slot, t, batch, hw, num_labels, seed_offset, out,
                                             mask_out, stream);
}

int pb200_gather_rows(const int64_t* pool, const int* slot, int64_t batch, int64_t hw, int64_t* out, void* stream) {
    PB_CHECK(batch >= 0 && batch <= 65535 && hw >= 0, "gather_rows: bad shape");
    if (batch == 0 || hw == 0) return 0;
    gather_rows_kernel<<<dim3(ceil_div(hw, 256), (unsigned)batch), 256, 0, (cudaStream_t)stream>>>(pool, slot, hw, out);
    PB_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
