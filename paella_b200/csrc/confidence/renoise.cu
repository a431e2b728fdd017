// Confidence-guided renoise: the renoise step of the sampling loop [ref/src/modules.py:277-283, Paella.add_noise] with the
// random mask replaced by each sample's least likely tokens (MaskGIT's choice rule), on the uniforms add_noise draws.
#include "confidence.h"

namespace pb {
// ------------------------------------------------------------------ confidence-guided renoise
// The renoise of a sampling step that replaces each sample's n least likely tokens instead of a random set (utils module
// docstring).  One CTA per sample b.  For each candidate token j (inside the region, all tokens without one):
//   u_j = the uniform add_noise draws for the token (same stream, same element, so every generator ends where add_noise leaves it)
//   k_j = logp_j + (tau_b * t_b) * g_j,  g_j = -logf(-logf(u_j))    (each operation rounded; u = 0 gives g = -inf)
// n = floor(fp32(t_b * N)), N the candidate count; the n smallest keys are renoised, ties to the lower index.  The keys live in
// shared memory as order-preserving 32-bit patterns (NaN -> 0, below every other key; non-candidates 0xffffffff, above every
// key); a radix select of four 8-bit passes finds the n-th smallest, and a block scan in index order resolves ties at it, so the
// result depends on no thread order.  A row with tau_b < 0 is add_noise's own rule (u <= t) and a row with t_b < 0 keeps its
// tokens: a mixed batch renoises in one launch.
constexpr int RN_THREADS = 512;
constexpr int RN_MAX_HW = PBC_RENOISE_MAX_HW;

__device__ __forceinline__ uint32_t renoise_order_key(float k) {
    const uint32_t b = __float_as_uint(k);
    return isnan(k) ? 0u : (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// x, logp, mask_out: [batch, hw] by sample; random_x, src, region, out: by slot (slot NULL = identity).  seed_off NULL: one
// stream s over batch * hw elements (sample b's token j is element b * hw + j, as add_noise_kernel); else sample b draws
// element j on its own (seed, offset) with the stride of s (as add_noise_per_sample_kernel).
__global__ void __launch_bounds__(RN_THREADS) renoise_confidence_kernel(
    const int64_t* __restrict__ x, const int64_t* __restrict__ random_x, const int64_t* __restrict__ src,
    const uint8_t* __restrict__ region, const int* __restrict__ slot, const float* __restrict__ logp, const float* __restrict__ t,
    const float* __restrict__ tau, int64_t hw, TorchPhilox s, const uint64_t* __restrict__ seed_off, int64_t* __restrict__ out,
    int64_t* __restrict__ mask_out) {
    extern __shared__ uint32_t rn_keys[];
    __shared__ uint32_t hist[256];
    __shared__ uint32_t warp_n[RN_THREADS / 32];
    __shared__ uint32_t sh_count, sh_prefix, sh_want;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t b = blockIdx.x;
    const int64_t dst = slot ? (int64_t)slot[b] : b;
    TorchPhilox sm = s;
    if (seed_off) {             // rng.cu's per-sample stream: sample b's (seed, offset), the stride of one sample's draw
        sm.seed = seed_off[2 * b];
        sm.offset4 = seed_off[2 * b + 1] >> 2;
    }
    const uint64_t e0 = seed_off ? 0 : (uint64_t)(b * hw);
    const float tb = t[b], taub = tau[b];
    const uint8_t* reg = region ? region + dst * hw : nullptr;
    auto uniform = [&](int64_t j) {
        const float u = u32_to_uniform(torch_philox_u32(sm, e0 + (uint64_t)j));
        return u == 1.0f ? 0.0f : u;
    };
    auto write = [&](int64_t j, bool gen, bool m) {
        out[dst * hw + j] = gen ? (m ? random_x[dst * hw + j] : x[b * hw + j]) : src[dst * hw + j];
        if (mask_out) mask_out[b * hw + j] = m ? 1 : 0;
    };
    if (taub < 0.f) {           // add_noise_per_sample_kernel's arithmetic
        for (int64_t j = tid; j < hw; j += RN_THREADS) {
            const bool gen = reg ? reg[j] != 0 : true;
            write(j, gen, gen && uniform(j) <= tb);
        }
        return;
    }
    if (tid == 0) sh_count = 0;
    __syncthreads();
    const float tt = __fmul_rn(taub, tb);
    uint32_t cnt = 0;
    for (int64_t j = tid; j < hw; j += RN_THREADS) {
        uint32_t k = 0xffffffffu;
        if (reg == nullptr || reg[j] != 0) {
            const float g = -logf(-logf(uniform(j)));
            k = renoise_order_key(__fadd_rn(logp[b * hw + j], __fmul_rn(tt, g)));
            ++cnt;
        }
        rn_keys[j] = k;
    }
    atomicAdd(&sh_count, cnt);
    __syncthreads();
    const uint32_t N = sh_count;
    uint32_t n = 0;
    if (tb >= 0.f) n = (uint32_t)fminf(floorf(__fmul_rn(tb, (float)N)), (float)N);
    // radix select: the n-th smallest key (prefix) and how many keys equal to it are taken (want)
    uint32_t prefix = 0, want = n;
    if (n > 0) {
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int i = tid; i < 256; i += RN_THREADS) hist[i] = 0;
            __syncthreads();
            const uint32_t high = shift == 24 ? 0u : 0xffffffffu << (shift + 8);
            for (int64_t j = tid; j < hw; j += RN_THREADS) {
                const uint32_t k = rn_keys[j];
                if ((k & high) == prefix) atomicAdd(&hist[(k >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (warp == 0) {
                uint32_t c[8], sum = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) { c[i] = hist[8 * lane + i]; sum += c[i]; }
                uint32_t incl = sum;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                }
                uint32_t before = incl - sum;
                if (before < want && want <= incl) {       // exactly one lane holds the n-th smallest
                    int d = 0;
                    while (before + c[d] < want) before += c[d++];
                    sh_prefix = prefix | ((uint32_t)(8 * lane + d) << shift);
                    sh_want = want - before;
                }
            }
            __syncthreads();
            prefix = sh_prefix;
            want = sh_want;
        }
    }
    // keys below the threshold are renoised, and the first `want` keys equal to it in index order
    const uint32_t thr = prefix;
    uint32_t eq_before = 0;
    for (int64_t base = 0; base < hw; base += RN_THREADS) {
        const int64_t j = base + tid;
        const uint32_t k = j < hw ? rn_keys[j] : 0xffffffffu;
        const bool eq = n > 0 && j < hw && k == thr;
        const uint32_t ballot = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) warp_n[warp] = __popc(ballot);
        __syncthreads();
        uint32_t rank = eq_before + __popc(ballot & ((1u << lane) - 1u)), total = 0;
        for (int w = 0; w < RN_THREADS / 32; ++w) {
            if (w < warp) rank += warp_n[w];
            total += warp_n[w];
        }
        __syncthreads();
        eq_before += total;
        if (j < hw) {
            const bool gen = reg ? reg[j] != 0 : true;
            write(j, gen, gen && n > 0 && (k < thr || (eq && rank < want)));
        }
    }
}

}  // namespace pb

extern "C" cudaError_t pbc_renoise_confidence_launch(const int64_t* x, const int64_t* random_x, const int64_t* src,
                                                     const uint8_t* region, const int* slot, const float* logp, const float* t,
                                                     const float* tau, int64_t batch, int64_t hw, pb::TorchPhilox s,
                                                     const uint64_t* seed_off, int64_t* out, int64_t* mask_out, cudaStream_t st) {
    using namespace pb;
    cudaError_t e = cudaFuncSetAttribute(renoise_confidence_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RN_MAX_HW * 4);
    if (e != cudaSuccess) return e;
    renoise_confidence_kernel<<<(unsigned)batch, RN_THREADS, (int)(hw * 4), st>>>(x, random_x, src, region, slot, logp, t, tau, hw,
                                                                                 s, seed_off, out, mask_out);
    return cudaGetLastError();
}
