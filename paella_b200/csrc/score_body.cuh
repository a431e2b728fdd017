// The body of the fused out_mapper + log-softmax kernels (score.cu's token_score_kernel, token_logprob.cu's
// token_logprob_kernel), one force-inlined template: each kernel lives in its own translation unit.
#pragma once
#include "gemm.cuh"
#include "score.cuh"

namespace pb {

constexpr int SC_BN = 128;
constexpr int SC_STAGES = 6;
constexpr int SC_MAX_KB = 4;                  // c_out <= 256
constexpr int SC_THREADS = 384;               // producer warpgroup + 2 MMA warpgroups
constexpr int SC_A_BYTES = 128 * 64 * 2;      // one k-block of the A tile
constexpr int SC_W_BYTES = SC_BN * 64 * 2;
constexpr int SC_SMEM = SC_MAX_KB * SC_A_BYTES + SC_STAGES * SC_W_BYTES + 1024 + 256;
constexpr float SC_LOG2E = 1.4426950408889634f;
constexpr float SC_LN2 = 0.6931471805599453f;

// (m, s) <- the log-sum-exp pair of (m, s) and (om, os), both in the log2 domain: s = sum 2^(x - m).  A side with no labels
// yet has m = -inf and s = 0 and contributes nothing (no inf - inf).
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
    const float mx = fmaxf(m, om);
    const float a = m == mx ? s : s * ptx::ex2_approx(m - mx);
    const float b = om == mx ? os : os * ptx::ex2_approx(om - mx);
    m = mx;
    s = a + b;
}

// The body of both kernels.  LOGP = false: token_score_kernel's statistics.  LOGP = true: the log-probability of the target
// under the tempered logits s = l * (1/T), one rounded product per logit, T of row r's sample r / hw (params [.][3], column 2,
// as the fused sampler's per-sample 1/T): logp_out[r] = s_y - lse(s); the sum, the arg-max and their registers drop out.
template <bool LOGP>
__device__ __forceinline__ void token_score_body(const CUtensorMap* tm_a, const CUtensorMap* tm_w, int R, int NL, int Kc,
                                                 float inv_nl, int hw, const float* __restrict__ params,
                                                 const int64_t* __restrict__ targets, float* __restrict__ nll_out,
                                                 float* __restrict__ smooth_out, int64_t* __restrict__ argmax_out) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t a_base = smem_base;
    const uint32_t w_base = smem_base + SC_MAX_KB * SC_A_BYTES;
    const uint32_t bar_base = w_base + SC_STAGES * SC_W_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (SC_STAGES + s); };
    const uint32_t a_bar = bar_base + 8u * (2 * SC_STAGES);

    const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
    const int lane = threadIdx.x & 31;
    const int n_kb = (Kc + 63) / 64;
    const int n_chunks = (NL + SC_BN - 1) / SC_BN;
    const int m_idx = blockIdx.x * 128;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(tm_a);
        ptx::prefetch_tensormap(tm_w);
        for (int s = 0; s < SC_STAGES; ++s) { ptx::mbar_init(full_bar(s), 1); ptx::mbar_init(empty_bar(s), 2); }
        ptx::mbar_init(a_bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x < 32 && ptx::elect_one()) {
            ptx::mbar_arrive_expect_tx(a_bar, n_kb * SC_A_BYTES);
            for (int kb = 0; kb < n_kb; ++kb) ptx::tma_load_2d(tm_a, a_bar, a_base + kb * SC_A_BYTES, kb * 64, m_idx);
            int stage = 0;
            uint32_t phase = 0;
            for (int ch = 0; ch < n_chunks; ++ch)
                for (int kb = 0; kb < n_kb; ++kb) {
                    ptx::mbar_wait(empty_bar(stage), phase ^ 1);
                    ptx::mbar_arrive_expect_tx(full_bar(stage), SC_W_BYTES);
                    ptx::tma_load_2d(tm_w, full_bar(stage), w_base + stage * SC_W_BYTES, kb * 64, ch * SC_BN);
                    if (++stage == SC_STAGES) { stage = 0; phase ^= 1; }
                }
        }
    } else {
        ptx::setmaxnreg_inc<232>();
        const int cw = wg - 1;                   // token rows [64 cw, 64 cw + 64) of the tile
        const int tid = threadIdx.x & 127;
        const int wq = tid >> 5;
        // this thread's two rows (wgmma fragment: rows 16 wq + lane/4 and + 8, column pairs 8n + 2 (lane % 4))
        const int row0 = m_idx + cw * 64 + wq * 16 + (lane >> 2);
        int64_t y[2] = {-1, -1};
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
            if (row0 + 8 * rr < R) y[rr] = targets[row0 + 8 * rr];
        // per row: running max m (log2 domain) and sum 2^(l log2e - m), sum of l, arg-max (value, label) and l_y
        float m[2] = {-INFINITY, -INFINITY}, s[2] = {0.f, 0.f}, sl[2] = {0.f, 0.f};
        float bv[2] = {-INFINITY, -INFINITY}, ly[2] = {NAN, NAN};
        int bi[2] = {0x7fffffff, 0x7fffffff};
        float inv_t[2] = {1.f, 1.f};
        if constexpr (LOGP) {
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
                if (row0 + 8 * rr < R) inv_t[rr] = params[3 * ((row0 + 8 * rr) / hw) + 2];
        }
        float acc[SC_BN / 2];
        ptx::mbar_wait(a_bar, 0);
        int stage = 0;
        uint32_t phase = 0;
        for (int ch = 0; ch < n_chunks; ++ch) {
            int prev = 0;
            for (int kb = 0; kb < n_kb; ++kb) {
                ptx::mbar_wait(full_bar(stage), phase);
                const uint64_t da = ptx::wgmma_desc_kmajor_sw128(a_base + kb * SC_A_BYTES + cw * (64 * 128));
                const uint64_t db = ptx::wgmma_desc_kmajor_sw128(w_base + stage * SC_W_BYTES);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) ptx::wgmma_m64n128k16(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
                ptx::wgmma_commit();
                if (kb > 0) {
                    ptx::wgmma_wait<1>();
                    if (tid == 0) ptx::mbar_arrive(empty_bar(prev));
                }
                prev = stage;
                if (++stage == SC_STAGES) { stage = 0; phase ^= 1; }
            }
            ptx::wgmma_wait<0>();
            if (tid == 0) ptx::mbar_arrive(empty_bar(prev));
            ptx::fence_regs(acc);
            // the chunk's maximum first, so each logit costs one exp
            float cm[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int i = 0; i < SC_BN / 2; ++i) {
                const int rr = (i >> 1) & 1;
                const int col = ch * SC_BN + (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
                if (col < NL) {
                    if constexpr (LOGP) acc[i] = __fmul_rn(acc[i], inv_t[rr]);
                    const float v = acc[i];
                    if constexpr (!LOGP)
                        if (v > bv[rr]) { bv[rr] = v; bi[rr] = col; }      // columns of a row arrive in increasing order
                    cm[rr] = fmaxf(cm[rr], v);
                    if constexpr (!LOGP) sl[rr] += v;
                    if ((int64_t)col == y[rr]) ly[rr] = v;
                }
            }
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const float nm = fmaxf(m[rr], cm[rr] * SC_LOG2E);
                if (nm > m[rr]) {
                    s[rr] = m[rr] == -INFINITY ? 0.f : s[rr] * ptx::ex2_approx(m[rr] - nm);
                    m[rr] = nm;
                }
            }
#pragma unroll
            for (int i = 0; i < SC_BN / 2; ++i) {
                const int rr = (i >> 1) & 1;
                const int col = ch * SC_BN + (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
                if (col < NL) s[rr] += ptx::ex2_approx(fmaf(acc[i], SC_LOG2E, -m[rr]));
            }
        }
        // combine the four threads of each row, in a fixed order
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                const float om = __shfl_xor_sync(0xffffffffu, m[rr], o), os = __shfl_xor_sync(0xffffffffu, s[rr], o);
                lse_merge(m[rr], s[rr], om, os);
                if constexpr (!LOGP) {
                    sl[rr] += __shfl_xor_sync(0xffffffffu, sl[rr], o);
                    const float ov = __shfl_xor_sync(0xffffffffu, bv[rr], o);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi[rr], o);
                    if (ov > bv[rr] || (ov == bv[rr] && oi < bi[rr])) { bv[rr] = ov; bi[rr] = oi; }
                }
                const float oy = __shfl_xor_sync(0xffffffffu, ly[rr], o);
                if (!isnan(oy)) ly[rr] = oy;          // at most one thread of the quad holds the target's column
            }
            const int row = row0 + 8 * rr;
            if ((lane & 3) == 0 && row < R) {
                const float lse = (m[rr] + __log2f(s[rr])) * SC_LN2;
                if constexpr (LOGP) {
                    // lse and the difference rounded as token_score_kernel rounds them: at 1/T = 1 this is -nll bit for bit
                    nll_out[row] = __fsub_rn(ly[rr], __fmul_rn(m[rr] + __log2f(s[rr]), SC_LN2));
                } else {
                    nll_out[row] = lse - ly[rr];
                    smooth_out[row] = lse - sl[rr] * inv_nl;
                    argmax_out[row] = bi[rr] == 0x7fffffff ? 0 : bi[rr];
                }
            }
        }
    }
}

}  // namespace pb
