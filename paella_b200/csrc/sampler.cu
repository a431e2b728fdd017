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

// PS (per-sample streams): the R rows are R / hw samples of hw rows; sample b draws on its own generator, (seed, philox
// offset) = seed_off[2b], seed_off[2b + 1], with rng's stride (the launch policy of ONE sample's draw), and element
// (row, col) of it is element (row - b hw) * NL + col of that draw -- what a batch-1 launch on that generator would use.
// skip (PS only, may be null): int32 [R / hw]; a sample with skip[b] != 0 does not draw this step and its rows of `out` are
// left as they are (a CTA whose rows all belong to such samples returns at once).
__device__ __forceinline__ void per_sample_stream(const uint64_t* __restrict__ seed_off, int b, TorchPhilox& s) {
    s.seed = seed_off[2 * b];
    s.offset4 = seed_off[2 * b + 1] >> 2;
}

// PP (per-sample parameters): row r of the launch belongs to sample r / phw, whose temperature is params[3 (r / phw) + 2] =
// 1.0f / (float)T_b (the (cfg, 1 - cfg) columns were applied by the pre-mix); the scalar instances read inv_t instead.
__device__ __forceinline__ float per_sample_inv_t(const float* __restrict__ params, int64_t row, int phw) {
    return params[3 * (row / phw) + 2];
}

// =====================================================================================================================
// Top-k / top-p truncation (TR instances, always with per-sample parameters).  A slot is one token row of the launch (the
// generic kernel's 128 rows, the shared kernel's 80 token columns).  With s_j = l_j * (1/T) the fp32 product (__fmul_rn: the
// same value in every pass) and key(s) the order-preserving 32-bit image of s:
//   top-k: tau_k = the k-th largest key (equal values counted separately); kept = {j : key_j >= tau_k};
//   top-p: W_j = floor(2^32 expf(s_j - m)) over the top-k kept set (m = the row maximum, expf the full-precision fp32 exp,
//          at most 2 ulp), tau_p = the largest key v with sum_{key_i >= v} W_i >= p * sum W_i (compared in fp64);
// and the draw keeps only labels with key >= tau = max(tau_k, tau_p).  The thresholds come from radix-select passes over the
// keys, 4 bits per pass (TR_LEVELS passes per search), each pass recomputing the out_mapper product from the same resident
// features and the same W tiles: per slot a count histogram and a fixed-point mass histogram in shared memory, summed with
// integer atomics, so the result depends on no thread or CTA order.  Passes: one for m (if any slot has p), one search (k, or p
// alone), a second search for the slots with both (top-p above tau_k), then the draw.
constexpr int TR_BINS = 16;
constexpr int TR_LEVELS = 8;
constexpr float TR_FIX = 4294967296.0f;          // 2^32: the mass quantum is 2^-32 of the row maximum's weight

template <int N>
struct TruncSmem {
    unsigned long long mass[N][TR_BINS];         // fixed-point mass per digit of the current level
    unsigned long long above_c[N], above_m[N];   // count / mass of the keys above the current prefix's bin
    double target[N];                            // mass target p * sum W (mass searches)
    uint4 pd[N];                                 // the pass's view of a slot: (lo, prefix, flags, m bits); flags 1 = in the
                                                 // search, 2 = accumulates mass
    unsigned int tau[N];                         // the threshold key (0 = keep every label); 16-byte aligned
    unsigned int cnt[N][TR_BINS];
    unsigned int prefix[N], lo[N], mkey[N];
    int mode[N], k[N];                           // mode: 1 = top-k, 2 = top-p, 3 = both
    float p[N];
    // the current pass, for the shared kernel's MMA warpgroups (read from here, not held in registers across the pass):
    // kind 0 = the draw, 1 = the maxima, 2 = a level; the level's prefix mask and digit shift
    int kind, shift;
    unsigned int mask;
};

__device__ __forceinline__ uint32_t tr_key(float s) {
    const uint32_t u = __float_as_uint(s + 0.0f);        // -0 -> +0: equal values, equal keys
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float tr_unkey(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// the pass's view of slot t for level L of search sr (0: k, or p alone; 1: p above tau_k)
template <int N>
__device__ __forceinline__ void tr_desc(TruncSmem<N>& ts, int t, int sr) {
    const int mode = ts.mode[t];
    const bool in = sr == 0 ? mode != 0 : mode == 3;
    ts.pd[t] = make_uint4(ts.lo[t], ts.prefix[t], (in ? 1u : 0u) | (in && (mode & 2) ? 2u : 0u), __float_as_uint(tr_unkey(ts.mkey[t])));
}

// slot t's (k, p) from the table (k <= 0 and p outside (0, 1) are off; k > NL is NL); returns its mode
template <int N>
__device__ __forceinline__ int tr_setup(TruncSmem<N>& ts, int t, bool valid, const int* __restrict__ trk, const float* __restrict__ trp,
                                        int64_t b, int NL) {
    const int k = valid ? trk[b] : 0;
    const float p = valid ? trp[b] : 1.0f;
    const int mode = (k > 0 ? 1 : 0) | (p > 0.0f && p < 1.0f ? 2 : 0);
    ts.mode[t] = mode;
    ts.k[t] = min(k, NL);
    ts.p[t] = p;
    ts.prefix[t] = ts.lo[t] = ts.tau[t] = ts.mkey[t] = 0;
    ts.above_c[t] = ts.above_m[t] = 0;
    ts.target[t] = 0.0;
#pragma unroll
    for (int d = 0; d < TR_BINS; ++d) { ts.cnt[t][d] = 0; ts.mass[t][d] = 0; }
    tr_desc(ts, t, 0);
    return mode;
}

// one label of a slot in a level pass: its key into the level's histograms if it lies in the slot's current bin
template <int N>
__device__ __forceinline__ void tr_add(TruncSmem<N>& ts, int t, float s, const uint4& pd, uint32_t mask, int shift) {
    const uint32_t key = tr_key(s);
    if ((pd.z & 1u) && key >= pd.x && ((key ^ pd.y) & mask) == 0) {
        const int d = (key >> shift) & (TR_BINS - 1);
        atomicAdd(&ts.cnt[t][d], 1u);
        if (pd.z & 2u) atomicAdd(&ts.mass[t][d], __float2ull_rz(expf(s - __uint_as_float(pd.w)) * TR_FIX));
    }
}

// after level L of search sr: slot t picks the largest digit whose cumulative count (k) or mass (p) reaches its target, and
// clears its histograms; at the last level the prefix is tau, and a slot with both k and p starts the top-p search above it
template <int N>
__device__ void tr_scan(TruncSmem<N>& ts, int t, int sr, int L) {
    const int mode = ts.mode[t];
    if (sr == 0 ? mode == 0 : mode != 3) return;
    const bool by_count = sr == 0 && (mode & 1);
    if (sr == 0 && !by_count && L == 0) {
        unsigned long long tot = 0;
#pragma unroll
        for (int d = 0; d < TR_BINS; ++d) tot += ts.mass[t][d];
        ts.target[t] = (double)ts.p[t] * (double)tot;
    }
    unsigned long long c = ts.above_c[t], w = ts.above_m[t];
    int sel = 0;
#pragma unroll 1
    for (int d = TR_BINS - 1; d >= 0; --d) {
        const unsigned long long nc = c + ts.cnt[t][d], nw = w + ts.mass[t][d];
        if (by_count ? nc >= (unsigned long long)ts.k[t] : (double)nw >= ts.target[t]) { sel = d; break; }
        c = nc;
        w = nw;
    }
    const unsigned long long wsel = ts.mass[t][sel];
#pragma unroll 1
    for (int d = 0; d < TR_BINS; ++d) { ts.cnt[t][d] = 0; ts.mass[t][d] = 0; }
    ts.above_c[t] = c;
    ts.above_m[t] = w;
    const uint32_t prefix = ts.prefix[t] | ((uint32_t)sel << (32 - 4 * (L + 1)));
    ts.prefix[t] = prefix;
    if (L == TR_LEVELS - 1) {
        ts.tau[t] = prefix;
        if (sr == 0 && mode == 3) {              // top-p over the top-k set: mass target p * sum_{key >= tau_k} W
            ts.target[t] = (double)ts.p[t] * (double)(w + wsel);
            ts.lo[t] = prefix;
            ts.prefix[t] = 0;
            ts.above_c[t] = ts.above_m[t] = 0;
        }
    }
}

// the view of pass `pass` (of n_sel selection passes, then the draw) in TruncSmem::kind / mask / shift
template <int N>
__device__ __forceinline__ void tr_pass_view(TruncSmem<N>& ts, int pass, int any_p, int n_sel) {
    const int j = pass - (any_p ? 1 : 0), L = j % TR_LEVELS;
    ts.kind = pass >= n_sel ? 0 : (any_p && pass == 0) ? 1 : 2;
    ts.mask = L <= 0 ? 0u : ~0u << (32 - 4 * L);
    ts.shift = 28 - 4 * L;
}

// the selection passes of a CTA: 1 for the row maxima if any slot has p, TR_LEVELS for the first search if any slot truncates,
// TR_LEVELS more if any slot has both
__device__ __forceinline__ int tr_passes(int any, int any_p, int any_both) {
    return (any_p ? 1 : 0) + (any ? TR_LEVELS : 0) + (any_both ? TR_LEVELS : 0);
}

constexpr int SMP_SMEM_TR = SMP_SMEM + (int)sizeof(TruncSmem<128>);

// TR (top-k / top-p, with PP): row r's (k, p) = trk[r / phw], trp[r / phw]; see TruncSmem.  The selection passes run the same
// chunk loop as the draw, the producer streaming the W tiles once per pass.
template <bool PS, bool PP, bool TR>
__global__ void __launch_bounds__(SMP_THREADS, 1)
fused_sampler_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w, int R, int NL,
                     int Kc, float inv_t, TorchPhilox rng, int hw, const uint64_t* __restrict__ seed_off,
                     const float* __restrict__ params, int phw, const int* __restrict__ skip, const int* __restrict__ trk,
                     const float* __restrict__ trp, int64_t* __restrict__ out) {
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
    if constexpr (PS) {
        // a tile whose rows all belong to samples that do not draw this step has nothing to write
        if (skip != nullptr) {
            const int b_last = (min(m_idx + 128, R) - 1) / hw;
            int b = m_idx / hw;
            while (b <= b_last && skip[b] != 0) ++b;
            if (b > b_last) return;
        }
    }

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tm_a);
        ptx::prefetch_tensormap(&tm_w);
        for (int s = 0; s < SMP_STAGES; ++s) { ptx::mbar_init(full_bar(s), 1); ptx::mbar_init(empty_bar(s), 2); }
        ptx::mbar_init(a_bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();
    // TR: per-row state, and the CTA's pass count (uniform: the producer streams W once per pass)
    auto tr_smem = [&]() -> TruncSmem<128>& {
        return *reinterpret_cast<TruncSmem<128>*>(smem_raw + (smem_base - smem_u32(smem_raw)) + (bar_base - smem_base) + 256);
    };
    int any_p = 0, any_both = 0, n_sel = 0;
    if constexpr (TR) {
        TruncSmem<128>& ts = tr_smem();
        int mode = 0;
        if (threadIdx.x < 128) {
            const int row = m_idx + threadIdx.x;
            const bool valid = row < R && !(PS && skip != nullptr && skip[row / hw] != 0);
            mode = tr_setup(ts, threadIdx.x, valid, trk, trp, row / phw, NL);
        }
        const int any = __syncthreads_or(mode != 0);
        any_p = __syncthreads_or(mode & 2);
        any_both = __syncthreads_or(mode == 3);
        n_sel = tr_passes(any, any_p, any_both);
    }

    if (wg == 0) {
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x < 32 && ptx::elect_one()) {
            ptx::mbar_arrive_expect_tx(a_bar, n_kb * SMP_A_BYTES);
            for (int kb = 0; kb < n_kb; ++kb) ptx::tma_load_2d(&tm_a, a_bar, a_base + kb * SMP_A_BYTES, kb * 64, m_idx);
            int stage = 0;
            uint32_t phase = 0;
            for (int pass = 0; pass <= n_sel; ++pass)
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
        TorchPhilox srng[2] = {rng, rng};
        uint64_t ebase[2] = {0, 0};
        if constexpr (PS) {
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int row = row0 + 8 * rr;
                if (row < R) {
                    const int b = row / hw;
                    per_sample_stream(seed_off, b, srng[rr]);
                    ebase[rr] = (uint64_t)(row - b * hw) * (uint64_t)NL;
                }
            }
        }
        float it[2] = {inv_t, inv_t};                // the two rows' 1/T
        if constexpr (PP) {
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
                if (row0 + 8 * rr < R) it[rr] = per_sample_inv_t(params, row0 + 8 * rr, phw);
        }
        float acc[SMP_BN / 2];
        ptx::mbar_wait(a_bar, 0);
        int stage = 0;
        uint32_t phase = 0;
        // the out_mapper product of label chunk ch for this warpgroup's 64 rows, into acc
        auto mma_chunk = [&]() {
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
        };
        uint32_t tau[2] = {0u, 0u};
        if constexpr (TR) {
            TruncSmem<128>& ts = tr_smem();
            const int t0 = cw * 64 + wq * 16 + (lane >> 2);          // the two rows' slots: t0, t0 + 8
            for (int pass = 0; pass < n_sel; ++pass) {
                const bool max_pass = any_p && pass == 0;
                const int j = pass - (any_p ? 1 : 0), sr = j / TR_LEVELS, L = j % TR_LEVELS;
                const uint32_t mask = L == 0 ? 0u : ~0u << (32 - 4 * L);
                const int shift = 28 - 4 * L;
                const uint4 pd[2] = {ts.pd[t0], ts.pd[t0 + 8]};
                float mx[2] = {-INFINITY, -INFINITY};
                for (int ch = 0; ch < n_chunks; ++ch) {
                    mma_chunk();
#pragma unroll
                    for (int i = 0; i < SMP_BN / 2; ++i) {
                        const int rr = (i >> 1) & 1;
                        const int col = ch * SMP_BN + (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
                        if (row0 + 8 * rr < R && col < NL) {
                            const float sv = __fmul_rn(acc[i], it[rr]);
                            if (max_pass) mx[rr] = fmaxf(mx[rr], sv);
                            else tr_add(ts, t0 + 8 * rr, sv, pd[rr], mask, shift);
                        }
                    }
                }
                if (max_pass) {
#pragma unroll
                    for (int rr = 0; rr < 2; ++rr) {
                        mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
                        mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
                        if ((lane & 3) == 0) ts.mkey[t0 + 8 * rr] = tr_key(mx[rr]);
                    }
                }
                ptx::bar_sync(1, 256);
                const int t = threadIdx.x - 128;
                if (t < 128) {
                    if (!max_pass) tr_scan(ts, t, sr, L);
                    const int jn = max_pass ? 0 : j + 1;              // the next level pass
                    if (jn < 2 * TR_LEVELS) tr_desc(ts, t, jn / TR_LEVELS);
                }
                ptx::bar_sync(1, 256);
            }
            tau[0] = ts.tau[t0];
            tau[1] = ts.tau[t0 + 8];
        }
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
                    const uint32_t bits = PS ? torch_philox_u32(srng[rr], ebase[rr] + (uint64_t)col)
                                             : torch_philox_u32(rng, (uint64_t)row * (uint64_t)NL + (uint64_t)col);
                    const float qv = torch_exponential1(u32_to_uniform(bits));
                    const float gum = fmaf(acc[i], PP ? it[rr] : inv_t, -__logf(qv));
                    const bool kept = !TR || tr_key(__fmul_rn(acc[i], it[rr])) >= tau[rr];     // excluded labels still draw
                    if (kept && gum > bv[rr]) { bv[rr] = gum; bi[rr] = col; }      // columns of a row arrive in increasing order
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
            if ((lane & 3) == 0 && row < R && !(PS && skip != nullptr && skip[row / hw] != 0)) out[row] = bi[rr];
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
constexpr int SH_SMEM_PP = SH_SMEM + SH_N * 4;     // + the per-column 1/T of a one-stream task
constexpr int SH_SMEM_TR = SH_SMEM_PP + (int)sizeof(TruncSmem<SH_N>);    // + the per-column truncation state

// PS: R / hw samples of hw rows, each with its own 4rs-row blocks (blocks_per_sample of them; the last one of a sample is
// partial and never straddles into the next sample's draw) and its own stream (see per_sample_stream).  The token tile comes
// through a 5-D map whose outermost coordinate is the sample; rows past a sample's end are loaded but never written.
// PP: per-sample 1/T (per_sample_inv_t).  With PS the CTA's rows are one sample's, so it is one load.  With one stream the
// four rows r + g rs of a Philox call can belong to different samples: the task's 80 token columns get their 1/T staged in
// shared memory once, and the epilogue reads them as one float4 per jj (its four g) -- not held in registers.
// TR (with PP): each of the 80 token columns has its own (k, p), as its 1/T, and its own truncation state and threshold in
// shared memory (TruncSmem); the draw reads the four g's thresholds of a jj as one uint4.
template <bool PS, bool PP, bool TR>
__global__ void __launch_bounds__(SH_THREADS, 1)
fused_sampler_shared_kernel(const __grid_constant__ CUtensorMap tm_f, const __grid_constant__ CUtensorMap tm_w, int R, int NL,
                            int Kc, int rs, int tasks_per_block, float inv_t, TorchPhilox rng, int hw, int blocks_per_sample,
                            const uint64_t* __restrict__ seed_off, const float* __restrict__ params, int phw,
                            const int* __restrict__ skip, const int* __restrict__ trk, const float* __restrict__ trp,
                            int64_t* __restrict__ out) {
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
    float* col_it = reinterpret_cast<float*>(tail + SH_RED_WARPS * SH_N * 8);   // [SH_N] (PP, one stream)
    TruncSmem<SH_N>& ts = *reinterpret_cast<TruncSmem<SH_N>*>(tail + SH_RED_WARPS * SH_N * 8 + SH_N * 4);   // (TR)

    const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
    const int lane = threadIdx.x & 31;
    const int n_kb = (Kc + 63) / 64;
    const int n_chunks = (NL + 127) / 128;
    const int sample = PS ? (int)(blockIdx.x / (blocks_per_sample * tasks_per_block)) : 0;
    const int task = blockIdx.x - sample * blocks_per_sample * tasks_per_block;
    const int blk = task / tasks_per_block;                            // 4rs-row block = Philox call index
    const int jj0 = (task - blk * tasks_per_block) * SH_JJ;
    if constexpr (PS) {
        if (skip != nullptr && skip[sample] != 0) return;      // the CTA's sample does not draw this step: no TMA, no write
    }

    if constexpr (PP && !PS) {
        if (threadIdx.x < SH_N) {                    // token column c = jj_local * 4 + g, as in the reduction below
            const int jj = jj0 + (int)threadIdx.x / 4, g = threadIdx.x & 3;
            const int64_t row = (int64_t)blk * 4 * rs + (int64_t)g * rs + jj;
            col_it[threadIdx.x] = (jj < rs && row < R) ? per_sample_inv_t(params, row, phw) : inv_t;
        }
    }
    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tm_f);
        ptx::prefetch_tensormap(&tm_w);
        for (int s = 0; s < SH_STAGES; ++s) { ptx::mbar_init(full_bar(s), 1); ptx::mbar_init(empty_bar(s), 2); }
        ptx::mbar_init(f_bar, 1);
        ptx::fence_barrier_init();
    }
    __syncthreads();
    int any_p = 0, n_sel = 0;
    if constexpr (TR) {
        int mode = 0;
        if (threadIdx.x < SH_N) {                    // token column c = jj_local * 4 + g
            const int jj = jj0 + (int)threadIdx.x / 4, g = threadIdx.x & 3;
            const int64_t row = (int64_t)blk * 4 * rs + (int64_t)g * rs + jj;      // within the sample (PS) or the launch
            const bool valid = jj < rs && row < (PS ? (int64_t)hw : (int64_t)R);
            mode = tr_setup(ts, threadIdx.x, valid, trk, trp, PS ? (int64_t)sample : row / phw, NL);
        }
        const int any = __syncthreads_or(mode != 0);
        any_p = __syncthreads_or(mode & 2);
        if (threadIdx.x == 0) tr_pass_view(ts, 0, any_p, any);     // n_sel > 0 exactly when any: pass 0's kind is settled
        n_sel = tr_passes(any, any_p, __syncthreads_or(mode == 3));
    }

    if (wg == 0) {
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x < 32 && ptx::elect_one()) {
            ptx::mbar_arrive_expect_tx(f_bar, n_kb * SH_F_BYTES);
            for (int kb = 0; kb < n_kb; ++kb) {
                if constexpr (PS) ptx::tma_load_5d(&tm_f, f_bar, f_base + kb * SH_F_BYTES, kb * 64, 0, jj0, blk, sample);
                else ptx::tma_load_4d(&tm_f, f_bar, f_base + kb * SH_F_BYTES, kb * 64, 0, jj0, blk);
            }
            int stage = 0;
            uint32_t phase = 0;
            for (int pass = 0; pass <= n_sel; ++pass)
            for (int ch = 0; ch < n_chunks; ++ch)
                for (int kb = 0; kb < n_kb; ++kb) {
                    ptx::mbar_wait(empty_bar(stage), phase ^ 1);
                    ptx::mbar_arrive_expect_tx(full_bar(stage), SH_W_BYTES);
                    ptx::tma_load_2d(&tm_w, full_bar(stage), w_base + stage * SH_W_BYTES, kb * 64, ch * 128);
                    if (++stage == SH_STAGES) { stage = 0; phase ^= 1; }
                }
        }
    } else {
        ptx::setmaxnreg_inc<232>();    // 128 x 56 + 256 x 224 = 64 K registers
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
        TorchPhilox srng = rng;
        if constexpr (PS) per_sample_stream(seed_off, sample, srng);
        float it_s = inv_t;
        if constexpr (PP && PS) it_s = params[3 * sample + 2];
        float acc[SH_N / 2];
        ptx::mbar_wait(f_bar, 0);
        int stage = 0;
        uint32_t phase = 0;
        // the out_mapper product of one 128-label chunk for this warpgroup's 64 labels and the task's 80 token columns, into acc
        auto mma_chunk = [&]() {
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
        };
        // after the swap below: v[g] = the logit of (label, token column 4 (2 n + (q >> 1)) + g)
        auto swap_halves = [&](int n, float (&v)[4]) {
            // fragment: acc[4n + {0,1}] = (label row lane/4, g = 2 (q & 1) + {0,1}), acc[4n + {2,3}] = (row + 8, same g)
            const float s0 = odd ? acc[4 * n + 0] : acc[4 * n + 2];
            const float s1 = odd ? acc[4 * n + 1] : acc[4 * n + 3];
            const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1);
            const float r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
            v[0] = odd ? r0 : acc[4 * n + 0];
            v[1] = odd ? r1 : acc[4 * n + 1];
            v[2] = odd ? acc[4 * n + 2] : r0;
            v[3] = odd ? acc[4 * n + 3] : r1;
        };
        // TR: passes 0 .. n_sel - 1 select (the column maxima in bv, then the level histograms), pass n_sel draws.  One wgmma
        // loop serves all of them and the pass's kind, mask and shift are read from shared memory, so the selection passes add
        // no live registers to the draw's (separate loops per pass kind made ptxas spill and serialise the wgmma)
        for (int pass = 0; pass <= n_sel; ++pass) {
            if (TR && pass == n_sel) {
                // the draw starts here: bv / bi (bv held the maxima) are not live across the selection passes
#pragma unroll
                for (int i = 0; i < SH_N / 2; ++i) { bv[i] = -INFINITY; bi[i] = 0x7fffffff; }
            }
            for (int ch = 0; ch < n_chunks; ++ch) {
                mma_chunk();
                const int kind = TR ? ts.kind : 0;
                const int label = ch * 128 + l;
#pragma unroll
                for (int n = 0; n < SH_N / 8; ++n) {
                    float v[4];
                    swap_halves(n, v);
                    if (label < NL) {
                        // the four g's 1/T: per column with one stream (staged in shared memory), else the sample's
                        auto col_inv_t = [&](float (&itg)[4]) {
                            if constexpr (PP && !PS) {
                                const float4 c4 = reinterpret_cast<const float4*>(col_it)[2 * n + (q >> 1)];
                                itg[0] = c4.x; itg[1] = c4.y; itg[2] = c4.z; itg[3] = c4.w;
                            }
                        };
                        float itg[4] = {it_s, it_s, it_s, it_s};
                        if (kind != 0) {                // s = l * (1/T), the fp32 product the draw's kept test sees
                            col_inv_t(itg);
                            const int c0 = (2 * n + (q >> 1)) * 4;
#pragma unroll
                            for (int g = 0; g < 4; ++g) {
                                const float sv = __fmul_rn(v[g], itg[g]);
                                if (kind == 1) bv[4 * n + g] = fmaxf(bv[4 * n + g], sv);
                                else tr_add(ts, c0 + g, sv, ts.pd[c0 + g], ts.mask, ts.shift);
                            }
                            continue;
                        }
                        const int jj = jj0 + 2 * n + (q >> 1);
                        const uint4 r4 = torch_philox_call(srng, (uint64_t)jj * (uint64_t)NL + (uint64_t)label, (uint64_t)blk);
                        const uint32_t bits[4] = {r4.x, r4.y, r4.z, r4.w};
                        col_inv_t(itg);
                        uint4 tau4 = make_uint4(0u, 0u, 0u, 0u);
                        if constexpr (TR) tau4 = reinterpret_cast<const uint4*>(ts.tau)[2 * n + (q >> 1)];
                        const uint32_t tau[4] = {tau4.x, tau4.y, tau4.z, tau4.w};
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            const float qv = torch_exponential1(u32_to_uniform(bits[g]));
                            const float gum = fmaf(v[g], PP ? itg[g] : inv_t, -__logf(qv));
                            const bool kept = !TR || tr_key(__fmul_rn(v[g], itg[g])) >= tau[g];    // excluded labels still draw
                            if (kept && gum > bv[4 * n + g]) { bv[4 * n + g] = gum; bi[4 * n + g] = label; }
                        }
                    }
                }
            }
            if (TR && pass < n_sel) {
                if (ts.kind == 1) {     // this warp's column maxima (every lane of a q >> 1 half holds its columns') to red_v
#pragma unroll
                    for (int i = 0; i < SH_N / 2; ++i) {
#pragma unroll
                        for (int o = 1; o <= 16; o <<= 1)
                            if (o != 2) bv[i] = fmaxf(bv[i], __shfl_xor_sync(0xffffffffu, bv[i], o));
                    }
#pragma unroll
                    for (int n = 0; n < SH_N / 8; ++n)
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            red_v[(cw * 4 + wq) * SH_N + (2 * n + (q >> 1)) * 4 + g] = bv[4 * n + g];
                            bv[4 * n + g] = -INFINITY;
                        }
                }
                ptx::bar_sync(1, 256);
                const int t = threadIdx.x - 128;
                if (t < SH_N) {
                    if (any_p && pass == 0) {
                        float mx = red_v[t];
                        for (int w = 1; w < SH_RED_WARPS; ++w) mx = fmaxf(mx, red_v[w * SH_N + t]);
                        ts.mkey[t] = tr_key(mx);
                        tr_desc(ts, t, 0);
                    } else {
                        const int j = pass - (any_p ? 1 : 0);
                        tr_scan(ts, t, j / TR_LEVELS, j % TR_LEVELS);
                        if (j + 1 < 2 * TR_LEVELS) tr_desc(ts, t, (j + 1) / TR_LEVELS);
                    }
                    if (t == 0) tr_pass_view(ts, pass + 1, any_p, n_sel);
                }
                ptx::bar_sync(1, 256);
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
            const int64_t row = (int64_t)blk * 4 * rs + (int64_t)g * rs + jj;      // within the sample (PS) or the launch
            if constexpr (PS) {
                if (jj < rs && row < hw) out[(int64_t)sample * hw + row] = besti;
            } else {
                if (jj < rs && row < R) out[row] = besti;
            }
        }
    }
}

int64_t fused_sampler_rows_padded(int64_t R, int NL) {
    TorchPhilox rng = make_torch_philox(0, 0, R * (int64_t)NL);
    if (NL <= 0 || rng.stride % (uint32_t)NL != 0) return R;
    const int64_t rs = rng.stride / NL;
    return (R + 4 * rs - 1) / (4 * rs) * (4 * rs);
}

// One launch over n_samp streams of hw rows each: n_samp == 1 with seed_off == nullptr is the single-stream draw (seed,
// offset) over all rows; otherwise seed_off is the device table of the per-sample streams.  Either way the kernel family
// and the Philox stride follow torch's launch policy for ONE stream's hw * NL elements.  params == nullptr: one 1/T, inv_t;
// otherwise the device table [R / phw][3] of per-sample parameters (PP instances).  trk / trp (with params): the per-sample
// truncation table (TR instances).
template <bool PS, bool PP, bool TR>
static void launch_shared(unsigned grid, const CUtensorMap& tf, const CUtensorMap& tw, int R, int NL, int Kc, int rs, int tpb,
                          float inv_t, TorchPhilox rng, int hw, int n_blocks, const uint64_t* seed_off, const float* params,
                          int phw, const int* skip, const int* trk, const float* trp, int64_t* out, cudaStream_t st) {
    fused_sampler_shared_kernel<PS, PP, TR><<<grid, SH_THREADS, TR ? SH_SMEM_TR : PP ? SH_SMEM_PP : SH_SMEM, st>>>(
        tf, tw, R, NL, Kc, rs, tpb, inv_t, rng, hw, n_blocks, seed_off, params, phw, skip, trk, trp, out);
}

template <bool PS, bool PP, bool TR>
static void launch_generic(unsigned grid, const CUtensorMap& ta, const CUtensorMap& tw, int R, int NL, int Kc, float inv_t,
                           TorchPhilox rng, int hw, const uint64_t* seed_off, const float* params, int phw, const int* skip,
                           const int* trk, const float* trp, int64_t* out, cudaStream_t st) {
    fused_sampler_kernel<PS, PP, TR><<<grid, SMP_THREADS, TR ? SMP_SMEM_TR : SMP_SMEM, st>>>(
        ta, tw, R, NL, Kc, inv_t, rng, hw, seed_off, params, phw, skip, trk, trp, out);
}

static int launch_sampler(const __half* a16, int64_t n_samp, int64_t hw, int Kc, const __half* w16, int NL, float inv_t,
                          uint64_t seed, uint64_t offset, const uint64_t* seed_off, const float* params, int64_t phw,
                          const int* skip, const int* trk, const float* trp, int64_t* out, cudaStream_t st) {
    const bool ps = seed_off != nullptr, pp = params != nullptr, tr = trk != nullptr;
    const int64_t R = n_samp * hw;
    TorchPhilox rng = make_torch_philox(seed, offset, hw * (int64_t)NL);
    {
        // shared-Philox path: needs stride % NL == 0 (rows of a lane group are whole rows).  The feature buffer must hold
        // (n_samp - 1) * hw + fused_sampler_rows_padded(hw, NL) rows (the caller's workspace does); rows past a stream's
        // end are never written to `out`.
        static const bool no_shared = getenv("PB200_SAMPLER_GENERIC") != nullptr;
        if (!no_shared && rng.stride % (uint32_t)NL == 0 && (int64_t)rng.stride / NL < (1 << 24)) {
            const int rs = (int)(rng.stride / NL);
            const int n_blocks = (int)((hw + 4 * (int64_t)rs - 1) / (4 * (int64_t)rs));
            const int tpb = (rs + SH_JJ - 1) / SH_JJ;
            static DeviceOnce attr2;
            if (attr2.first()) {
                PB_CUDA(cudaFuncSetAttribute(fused_sampler_shared_kernel<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_SMEM));
                PB_CUDA(cudaFuncSetAttribute(fused_sampler_shared_kernel<true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_SMEM));
                PB_CUDA(cudaFuncSetAttribute(fused_sampler_shared_kernel<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_SMEM_PP));
                PB_CUDA(cudaFuncSetAttribute(fused_sampler_shared_kernel<true, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_SMEM_PP));
                PB_CUDA(cudaFuncSetAttribute(fused_sampler_shared_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_SMEM_TR));
                PB_CUDA(cudaFuncSetAttribute(fused_sampler_shared_kernel<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_SMEM_TR));
            }
            ProfScope prof("fused_sampler", 2.0 * (double)R * (double)NL * (double)Kc, st);
            CUtensorMap tf, tw;
            const int64_t dims[5] = {Kc, 4, rs, n_blocks, n_samp};
            const int64_t strides[4] = {(int64_t)rs * Kc * 2, (int64_t)Kc * 2, 4 * (int64_t)rs * Kc * 2, hw * Kc * 2};
            const int box[5] = {64, 4, SH_JJ, 1, 1};
            PB_TRY(make_tmap_f16_nd(&tf, a16, ps ? 5 : 4, dims, strides, box));
            PB_TRY(make_tmap_f16_2d(&tw, w16, NL, Kc, Kc, 128));
            const int64_t grid = n_samp * n_blocks * tpb;
            PB_CHECK(grid < (1ll << 31), "fused sampler: %lld CTAs", (long long)grid);
            auto* fn = tr ? (ps ? launch_shared<true, true, true> : launch_shared<false, true, true>)
                          : ps ? (pp ? launch_shared<true, true, false> : launch_shared<true, false, false>)
                               : (pp ? launch_shared<false, true, false> : launch_shared<false, false, false>);
            fn((unsigned)grid, tf, tw, (int)R, NL, Kc, rs, tpb, inv_t, rng, (int)hw, n_blocks, seed_off, params, (int)phw, skip, trk, trp,
               out, st);
            PB_LAUNCH_CHECK();
            return 0;
        }
    }
    static DeviceOnce attr_set;
    if (attr_set.first()) {
        PB_CUDA(cudaFuncSetAttribute(fused_sampler_kernel<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM));
        PB_CUDA(cudaFuncSetAttribute(fused_sampler_kernel<true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM));
        PB_CUDA(cudaFuncSetAttribute(fused_sampler_kernel<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM));
        PB_CUDA(cudaFuncSetAttribute(fused_sampler_kernel<true, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM));
        PB_CUDA(cudaFuncSetAttribute(fused_sampler_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM_TR));
        PB_CUDA(cudaFuncSetAttribute(fused_sampler_kernel<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMP_SMEM_TR));
    }
    ProfScope prof("fused_sampler", 2.0 * (double)R * (double)NL * (double)Kc, st);
    CUtensorMap ta, tw;
    PB_TRY(make_tmap_f16_2d(&ta, a16, R, Kc, Kc, 128));
    PB_TRY(make_tmap_f16_2d(&tw, w16, NL, Kc, Kc, SMP_BN));
    auto* fn = tr ? (ps ? launch_generic<true, true, true> : launch_generic<false, true, true>)
                  : ps ? (pp ? launch_generic<true, true, false> : launch_generic<true, false, false>)
                       : (pp ? launch_generic<false, true, false> : launch_generic<false, false, false>);
    fn((unsigned)ceil_div(R, 128), ta, tw, (int)R, NL, Kc, inv_t, rng, (int)hw, seed_off, params, (int)phw, skip, trk, trp, out, st);
    PB_LAUNCH_CHECK();
    return 0;
}

int launch_fused_sampler(const __half* a16, int64_t R, int Kc, const __half* w16, int NL, float inv_t, uint64_t seed,
                         uint64_t offset, int64_t* out, cudaStream_t st) {
    PB_CHECK(Kc % 8 == 0 && Kc <= 64 * SMP_MAX_KB, "fused sampler: c_out=%d unsupported (<= %d, multiple of 8)", Kc, 64 * SMP_MAX_KB);
    PB_CHECK(R * (int64_t)NL < (1ll << 31), "fused sampler: rows*labels >= 2^31 would split the torch kernel (unsupported)");
    PB_CHECK(offset % 4 == 0, "philox offset must be a multiple of 4");
    if (R == 0) return 0;
    return launch_sampler(a16, 1, R, Kc, w16, NL, inv_t, seed, offset, nullptr, nullptr, 1, nullptr, nullptr, nullptr, out, st);
}

int launch_fused_sampler_per_sample(const __half* a16, int64_t n_samp, int64_t hw, int Kc, const __half* w16, int NL,
                                    float inv_t, const uint64_t* seed_off, int64_t* out, cudaStream_t st) {
    PB_CHECK(seed_off != nullptr, "fused sampler: per-sample (seed, offset) table is NULL");
    return launch_fused_sampler_params(a16, n_samp, hw, Kc, w16, NL, inv_t, nullptr, 0, 0, seed_off, out, st);
}

int launch_fused_sampler_params(const __half* a16, int64_t n_samp, int64_t hw, int Kc, const __half* w16, int NL, float inv_t,
                                const float* params, uint64_t seed, uint64_t offset, const uint64_t* seed_off, int64_t* out,
                                cudaStream_t st, const int* skip, const int* top_k, const float* top_p) {
    PB_CHECK(skip == nullptr || seed_off != nullptr, "fused sampler: a skip table needs per-sample streams");
    PB_CHECK((top_k == nullptr) == (top_p == nullptr), "fused sampler: the truncation table needs both top_k and top_p");
    PB_CHECK(top_k == nullptr || params != nullptr, "fused sampler: a truncation table needs the per-sample parameter table");
    PB_CHECK(Kc % 8 == 0 && Kc <= 64 * SMP_MAX_KB, "fused sampler: c_out=%d unsupported (<= %d, multiple of 8)", Kc, 64 * SMP_MAX_KB);
    PB_CHECK(n_samp * hw < (1ll << 31), "fused sampler: %lld rows", (long long)(n_samp * hw));
    if (seed_off != nullptr) {
        PB_CHECK(hw * (int64_t)NL <= (1ll << 29),
                 "fused sampler: a per-sample draw of %lld elements (hw*labels > 2^29) would split the torch kernel (unsupported)",
                 (long long)(hw * (int64_t)NL));
    } else {
        PB_CHECK(n_samp * hw * (int64_t)NL < (1ll << 31),
                 "fused sampler: rows*labels >= 2^31 would split the torch kernel (unsupported)");
        PB_CHECK(offset % 4 == 0, "philox offset must be a multiple of 4");
    }
    if (n_samp == 0 || hw == 0) return 0;
    if (seed_off != nullptr)          // one stream per sample: a launch "sample" is a parameter sample
        return launch_sampler(a16, n_samp, hw, Kc, w16, NL, inv_t, 0, 0, seed_off, params, hw, skip, top_k, top_p, out, st);
    return launch_sampler(a16, 1, n_samp * hw, Kc, w16, NL, inv_t, seed, offset, nullptr, params, hw, nullptr, top_k, top_p, out, st);
}

}  // namespace pb
