// Fused out_mapper GEMM + temperature + multinomial draw: logits never reach HBM.
// Replaces ref/src/modules.py:184-187 (out_mapper 1x1 conv, 256 -> 8192) and ref/src/utils.py:45-50
// (CFG mix, /T, softmax, permute+reshape copy, torch.multinomial) — ~0.74 GB of HBM traffic per image-step in
// the reference, ~1 MB here (SURVEY.md §8d).
//
// The classifier-free-guidance mix is linear, so it is applied to the 256-wide LayerNorm'd features BEFORE the
// GEMM (one GEMM instead of two).  The draw is Gumbel-max in the log domain on torch's own random stream:
//     token = argmax_k ( l_k / T  -  log q_k ),   q_k = the Exp(1) variate torch.multinomial's
//                                                  exponential_() would hand to element (row, k)
// which equals argmax_k softmax(l/T)_k / q_k (what torch computes) up to fp32 rounding of near-ties.
//
// One CTA per 128 token rows, 384 threads:
//   warpgroup 0     TMA: the 128 x c_out A tile once (resident), then W tiles [128 labels x 64] through a 6-deep ring
//   warpgroups 1,2  wgmma m64n128k16 for 64 token rows each (accumulators in registers), then per element Philox4x32-10 and
//                   a running arg-max per row in registers; the quad of threads sharing a row is reduced at the end
#include <cstdlib>

#include "gemm.cuh"
#include "sampler.cuh"

namespace pb {

constexpr int SMP_BN = 128;
constexpr int SMP_STAGES = 6;
constexpr int SMP_MAX_KB = 4;                 // c_out <= 256
constexpr int SMP_THREADS = 384;              // producer warpgroup + 2 MMA warpgroups
constexpr int SMP_A_BYTES = 128 * 64 * 2;     // one k-block of the A tile
constexpr int SMP_W_BYTES = SMP_BN * 64 * 2;
constexpr int SMP_SMEM = SMP_MAX_KB * SMP_A_BYTES + SMP_STAGES * SMP_W_BYTES + 1024 + 256;

// keeps (v, i) if it wins: larger value, or equal value and smaller label (torch's first maximum)
__device__ __forceinline__ void argmax_merge(float& bv, int& bi, float ov, int oi) {
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
}

__global__ void __launch_bounds__(SMP_THREADS, 1)
fused_sampler_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w, int R, int NL,
                     int Kc, float inv_t, TorchPhilox rng, int64_t* __restrict__ out) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t a_base = smem_base;
    const uint32_t w_base = smem_base + SMP_MAX_KB * SMP_A_BYTES;
    const uint32_t bar_base = w_base + SMP_STAGES * SMP_W_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (SMP_STAGES + s); };
    const uint32_t a_bar = bar_base + 8u * (2 * SMP_STAGES);

    const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
    const int lane = threadIdx.x & 31;
    const int n_kb = (Kc + 63) / 64;
    const int n_chunks = (NL + SMP_BN - 1) / SMP_BN;
    const int m_idx = blockIdx.x * 128;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tm_a);
        ptx::prefetch_tensormap(&tm_w);
        for (int s = 0; s < SMP_STAGES; ++s) { ptx::mbar_init(full_bar(s), 1); ptx::mbar_init(empty_bar(s), 2); }
        ptx::mbar_init(a_bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x < 32 && ptx::elect_one()) {
            ptx::mbar_arrive_expect_tx(a_bar, n_kb * SMP_A_BYTES);
            for (int kb = 0; kb < n_kb; ++kb) ptx::tma_load_2d(&tm_a, a_bar, a_base + kb * SMP_A_BYTES, kb * 64, m_idx);
            int stage = 0;
            uint32_t phase = 0;
            for (int ch = 0; ch < n_chunks; ++ch)
                for (int kb = 0; kb < n_kb; ++kb) {
                    ptx::mbar_wait(empty_bar(stage), phase ^ 1);
                    ptx::mbar_arrive_expect_tx(full_bar(stage), SMP_W_BYTES);
                    ptx::tma_load_2d(&tm_w, full_bar(stage), w_base + stage * SMP_W_BYTES, kb * 64, ch * SMP_BN);
                    if (++stage == SMP_STAGES) { stage = 0; phase ^= 1; }
                }
        }
    } else {
        ptx::setmaxnreg_inc<232>();
        const int cw = wg - 1;                   // token rows [64 cw, 64 cw + 64) of the tile
        const int tid = threadIdx.x & 127;
        const int wq = tid >> 5;
        // this thread's two rows (wgmma fragment: rows 16 wq + lane/4 and + 8, column pairs 8n + 2 (lane % 4))
        const int row0 = m_idx + cw * 64 + wq * 16 + (lane >> 2);
        float bv[2] = {-INFINITY, -INFINITY};
        int bi[2] = {0x7fffffff, 0x7fffffff};
        float acc[SMP_BN / 2];
        ptx::mbar_wait(a_bar, 0);
        int stage = 0;
        uint32_t phase = 0;
        for (int ch = 0; ch < n_chunks; ++ch) {
            int prev = 0;
            for (int kb = 0; kb < n_kb; ++kb) {
                ptx::mbar_wait(full_bar(stage), phase);
                const uint64_t da = ptx::wgmma_desc_kmajor_sw128(a_base + kb * SMP_A_BYTES + cw * (64 * 128));
                const uint64_t db = ptx::wgmma_desc_kmajor_sw128(w_base + stage * SMP_W_BYTES);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) ptx::wgmma_m64n128k16(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
                ptx::wgmma_commit();
                if (kb > 0) {
                    ptx::wgmma_wait<1>();
                    if (tid == 0) ptx::mbar_arrive(empty_bar(prev));
                }
                prev = stage;
                if (++stage == SMP_STAGES) { stage = 0; phase ^= 1; }
            }
            ptx::wgmma_wait<0>();
            if (tid == 0) ptx::mbar_arrive(empty_bar(prev));
            ptx::fence_regs(acc);
#pragma unroll
            for (int i = 0; i < SMP_BN / 2; ++i) {
                const int rr = (i >> 1) & 1;
                const int row = row0 + 8 * rr;
                const int col = ch * SMP_BN + (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
                if (row < R && col < NL) {
                    const float qv = torch_exponential1(u32_to_uniform(torch_philox_u32(rng, (uint64_t)row * (uint64_t)NL + (uint64_t)col)));
                    const float gum = fmaf(acc[i], inv_t, -__logf(qv));
                    if (gum > bv[rr]) { bv[rr] = gum; bi[rr] = col; }      // columns of a row arrive in increasing order
                }
            }
        }
        // combine the four threads of each row
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1)
                argmax_merge(bv[rr], bi[rr], __shfl_xor_sync(0xffffffffu, bv[rr], o), __shfl_xor_sync(0xffffffffu, bi[rr], o));
            const int row = row0 + 8 * rr;
            if ((lane & 3) == 0 && row < R) out[row] = bi[rr];
        }
    }
}

// =====================================================================================================================
// Shared-Philox variant.  torch's generator hands element (row, label) the lane (row / rs) % 4 of curand4 call number
// row / (4 rs) of thread (row % rs) * NL + label, rs = stride / NL (33 on a 132-SM H100 for 8192 labels): the four rows
// r, r+rs, r+2rs, r+3rs of a 4rs-row block share ONE Philox4x32-10 evaluation per label.  To use all four outputs in
// one thread the product is computed TRANSPOSED — D[label, token] = W[labels, K] . F[tokens, K]^T — with the token
// tile ordered (jj, g) -> row 4rs*i + rs*g + jj0 + jj (a 4-D TMA box, g innermost).  Each MMA warpgroup takes 64 labels of a
// 128-label chunk (wgmma m64n80k16); in the fragment a thread holds two of the four g of a (label, jj) pair, so neighbouring
// threads swap halves: afterwards a thread owns one label and all four g of 10 jj = 10 Philox calls for 40 logits, keeps a
// running arg-max per token column over the 64 chunks in registers, and the labels are reduced once at the end.
constexpr int SH_JJ = 20;                      // jj slots per task
constexpr int SH_N = 4 * SH_JJ;                // token columns per MMA tile (wgmma N = 80)
constexpr int SH_THREADS = 384;
constexpr int SH_STAGES = 6;
constexpr int SH_F_BYTES = SH_N * 128;         // one k-block of the token tile
constexpr int SH_W_BYTES = 128 * 128;          // 128 labels x 64 halves
constexpr int SH_RED_WARPS = 8;                // MMA warps, one reduction row each
constexpr int SH_SMEM = SMP_MAX_KB * SH_F_BYTES + SH_STAGES * SH_W_BYTES + 1024 + 256 + SH_RED_WARPS * SH_N * 8;

__global__ void __launch_bounds__(SH_THREADS, 1)
fused_sampler_shared_kernel(const __grid_constant__ CUtensorMap tm_f, const __grid_constant__ CUtensorMap tm_w, int R, int NL,
                            int Kc, int rs, int tasks_per_block, float inv_t, TorchPhilox rng, int64_t* __restrict__ out) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    const uint32_t f_base = smem_base;
    const uint32_t w_base = smem_base + SMP_MAX_KB * SH_F_BYTES;
    const uint32_t bar_base = w_base + SH_STAGES * SH_W_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (SH_STAGES + s); };
    const uint32_t f_bar = bar_base + 8u * (2 * SH_STAGES);
    uint8_t* tail = smem_gen + (bar_base - smem_base) + 256;
    float* red_v = reinterpret_cast<float*>(tail);                    // [8 warps][SH_N]
    int* red_i = reinterpret_cast<int*>(tail + SH_RED_WARPS * SH_N * 4);

    const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
    const int lane = threadIdx.x & 31;
    const int n_kb = (Kc + 63) / 64;
    const int n_chunks = (NL + 127) / 128;
    const int blk = blockIdx.x / tasks_per_block;                      // 4rs-row block = Philox call index
    const int jj0 = (blockIdx.x - blk * tasks_per_block) * SH_JJ;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tm_f);
        ptx::prefetch_tensormap(&tm_w);
        for (int s = 0; s < SH_STAGES; ++s) { ptx::mbar_init(full_bar(s), 1); ptx::mbar_init(empty_bar(s), 2); }
        ptx::mbar_init(f_bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x < 32 && ptx::elect_one()) {
            ptx::mbar_arrive_expect_tx(f_bar, n_kb * SH_F_BYTES);
            for (int kb = 0; kb < n_kb; ++kb) ptx::tma_load_4d(&tm_f, f_bar, f_base + kb * SH_F_BYTES, kb * 64, 0, jj0, blk);
            int stage = 0;
            uint32_t phase = 0;
            for (int ch = 0; ch < n_chunks; ++ch)
                for (int kb = 0; kb < n_kb; ++kb) {
                    ptx::mbar_wait(empty_bar(stage), phase ^ 1);
                    ptx::mbar_arrive_expect_tx(full_bar(stage), SH_W_BYTES);
                    ptx::tma_load_2d(&tm_w, full_bar(stage), w_base + stage * SH_W_BYTES, kb * 64, ch * 128);
                    if (++stage == SH_STAGES) { stage = 0; phase ^= 1; }
                }
        }
    } else {
        ptx::setmaxnreg_inc<232>();
        const int cw = wg - 1;                       // labels [64 cw, 64 cw + 64) of each chunk
        const int tid = threadIdx.x & 127;
        const int wq = tid >> 5;
        const int q = lane & 3;
        const bool odd = (q & 1) != 0;
        // after the swap: this thread's label of the chunk, and jj = jj0 + 2 n + (q >> 1) for n = 0..9, all four g
        const int l = cw * 64 + wq * 16 + (lane >> 2) + (odd ? 8 : 0);
        float bv[SH_N / 2];
        int bi[SH_N / 2];
#pragma unroll
        for (int i = 0; i < SH_N / 2; ++i) { bv[i] = -INFINITY; bi[i] = 0x7fffffff; }
        float acc[SH_N / 2];
        ptx::mbar_wait(f_bar, 0);
        int stage = 0;
        uint32_t phase = 0;
        for (int ch = 0; ch < n_chunks; ++ch) {
            int prev = 0;
            for (int kb = 0; kb < n_kb; ++kb) {
                ptx::mbar_wait(full_bar(stage), phase);
                const uint64_t da = ptx::wgmma_desc_kmajor_sw128(w_base + stage * SH_W_BYTES + cw * (64 * 128));   // labels = M
                const uint64_t db = ptx::wgmma_desc_kmajor_sw128(f_base + kb * SH_F_BYTES);                        // tokens = N
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) ptx::wgmma_m64n80k16(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
                ptx::wgmma_commit();
                if (kb > 0) {
                    ptx::wgmma_wait<1>();
                    if (tid == 0) ptx::mbar_arrive(empty_bar(prev));
                }
                prev = stage;
                if (++stage == SH_STAGES) { stage = 0; phase ^= 1; }
            }
            ptx::wgmma_wait<0>();
            if (tid == 0) ptx::mbar_arrive(empty_bar(prev));
            ptx::fence_regs(acc);
            const int label = ch * 128 + l;
#pragma unroll
            for (int n = 0; n < SH_N / 8; ++n) {
                // fragment: acc[4n + {0,1}] = (label row lane/4, g = 2 (q & 1) + {0,1}), acc[4n + {2,3}] = (row + 8, same g)
                const float s0 = odd ? acc[4 * n + 0] : acc[4 * n + 2];
                const float s1 = odd ? acc[4 * n + 1] : acc[4 * n + 3];
                const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1);
                const float r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
                float v[4];
                v[0] = odd ? r0 : acc[4 * n + 0];
                v[1] = odd ? r1 : acc[4 * n + 1];
                v[2] = odd ? acc[4 * n + 2] : r0;
                v[3] = odd ? acc[4 * n + 3] : r1;
                if (label < NL) {
                    const int jj = jj0 + 2 * n + (q >> 1);
                    const uint4 r4 = torch_philox_call(rng, (uint64_t)jj * (uint64_t)NL + (uint64_t)label, (uint64_t)blk);
                    const uint32_t bits[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const float qv = torch_exponential1(u32_to_uniform(bits[g]));
                        const float gum = fmaf(v[g], inv_t, -__logf(qv));
                        if (gum > bv[4 * n + g]) { bv[4 * n + g] = gum; bi[4 * n + g] = label; }
                    }
                }
            }
        }
        // reduce over the labels of this warp (lanes with the same q >> 1 hold the same token columns), then over the 8 warps
#pragma unroll
        for (int i = 0; i < SH_N / 2; ++i) {
#pragma unroll
            for (int o = 1; o <= 16; o <<= 1) {
                if (o == 2) continue;
                argmax_merge(bv[i], bi[i], __shfl_xor_sync(0xffffffffu, bv[i], o), __shfl_xor_sync(0xffffffffu, bi[i], o));
            }
        }
        const int w8 = cw * 4 + wq;
        if (lane == 0 || lane == 2) {
#pragma unroll
            for (int n = 0; n < SH_N / 8; ++n)
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const int c = (2 * n + (q >> 1)) * 4 + g;       // token column = jj_local * 4 + g
                    red_v[w8 * SH_N + c] = bv[4 * n + g];
                    red_i[w8 * SH_N + c] = bi[4 * n + g];
                }
        }
        ptx::bar_sync(1, 256);
        const int t = threadIdx.x - 128;
        if (t < SH_N) {
            float best = red_v[t];
            int besti = red_i[t];
#pragma unroll
            for (int w = 1; w < SH_RED_WARPS; ++w) argmax_merge(best, besti, red_v[w * SH_N + t], red_i[w * SH_N + t]);
            const int jj = jj0 + t / 4, g = t & 3;
            const int64_t row = (int64_t)blk * 4 * rs + (int64_t)g * rs + jj;
            if (jj < rs && row < R) out[row] = besti;
        }
    }
}

int64_t fused_sampler_rows_padded(int64_t R, int NL) {
    TorchPhilox rng = make_torch_philox(0, 0, R * (int64_t)NL);
    if (NL <= 0 || rng.stride % (uint32_t)NL != 0) return R;
    const int64_t rs = rng.stride / NL;
    return (R + 4 * rs - 1) / (4 * rs) * (4 * rs);
}

int launch_fused_sampler(const __half* a16, int64_t R, int Kc, const __half* w16, int NL, float inv_t, uint64_t seed,
                         uint64_t offset, int64_t* out, cudaStream_t st) {
    PB_CHECK(Kc % 8 == 0 && Kc <= 64 * SMP_MAX_KB, "fused sampler: c_out=%d unsupported (<= %d, multiple of 8)", Kc, 64 * SMP_MAX_KB);
    PB_CHECK(R * (int64_t)NL < (1ll << 31), "fused sampler: rows*labels >= 2^31 would split the torch kernel (unsupported)");
    PB_CHECK(offset % 4 == 0, "philox offset must be a multiple of 4");
    if (R == 0) return 0;
    {
        // shared-Philox path: needs stride % NL == 0 (rows of a lane group are whole rows).  The feature buffer must hold
        // fused_sampler_rows_padded(R, NL) rows (the caller's workspace does); rows >= R are never written to `out`.
        TorchPhilox rng = make_torch_philox(seed, offset, R * (int64_t)NL);
        static const bool no_shared = getenv("PB200_SAMPLER_GENERIC") != nullptr;
        if (!no_shared && rng.stride % (uint32_t)NL == 0 && (int64_t)rng.stride / NL < (1 << 24)) {
            const int rs = (int)(rng.stride / NL);
            const int n_blocks = (int)((R + 4 * (int64_t)rs - 1) / (4 * (int64_t)rs));
            const int tpb = (rs + SH_JJ - 1) / SH_JJ;
            static DeviceOnce attr2;
            if (attr2.first()) {
                PB_CUDA(cudaFuncSetAttribute(fused_sampler_shared_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_SMEM));
    }
            ProfScope prof("fused_sampler", 2.0 * (double)R * (double)NL * (double)Kc, st);
            CUtensorMap tf, tw;
            const int64_t dims[4] = {Kc, 4, rs, n_blocks};
            const int64_t strides[3] = {(int64_t)rs * Kc * 2, (int64_t)Kc * 2, 4 * (int64_t)rs * Kc * 2};
            const int box[4] = {64, 4, SH_JJ, 1};
            PB_TRY(make_tmap_f16_nd(&tf, a16, 4, dims, strides, box));
            PB_TRY(make_tmap_f16_2d(&tw, w16, NL, Kc, Kc, 128));
            fused_sampler_shared_kernel<<<n_blocks * tpb, SH_THREADS, SH_SMEM, st>>>(tf, tw, (int)R, NL, Kc, rs, tpb, inv_t, rng, out);
            PB_LAUNCH_CHECK();
            return 0;
        }
    }
    static DeviceOnce attr_set;
    if (attr_set.first()) {
        PB_CUDA(cudaFuncSetAttribute(fused_sampler_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM));
    }
    ProfScope prof("fused_sampler", 2.0 * (double)R * (double)NL * (double)Kc, st);
    CUtensorMap ta, tw;
    PB_TRY(make_tmap_f16_2d(&ta, a16, R, Kc, Kc, 128));
    PB_TRY(make_tmap_f16_2d(&tw, w16, NL, Kc, Kc, SMP_BN));
    TorchPhilox rng = make_torch_philox(seed, offset, R * (int64_t)NL);
    fused_sampler_kernel<<<ceil_div(R, 128), SMP_THREADS, SMP_SMEM, st>>>(ta, tw, (int)R, NL, Kc, inv_t, rng, out);
    PB_LAUNCH_CHECK();
    return 0;
}

}  // namespace pb
