// wgmma + TMA attention core for head_dim 80 (the reference model's 1280 / 16): every query count and key count of the
// workloads, varlen conditioning (kv_len), shared conditioning slots (kv_slot) and post-softmax attn_weights.
//
// One CTA (one warpgroup, 128 threads) per (64 queries, head, sample); warp w owns query rows [16 w, 16 w + 16).
//   TMA       Q once; K and V of 64-key chunks (the sample's self keys from qkv, then its conditioning keys from ckv) into a
//             2-stage ring on full mbarriers.  head_dim 80 = a 64-wide SWIZZLE_128B box + a 16-wide SWIZZLE_32B box for Q and
//             K (the K-major operands of S = Q K^T); V lands as it lies in memory and is transposed once per chunk into a
//             SWIZZLE_128B [80 dims x 64 keys] tile, the K-major B operand of O += P V.
//   wgmma     S[64 x 64] = Q K^T: m64n64k16 x 5 from shared memory; O[64 x 80] += P V: m64n80k16 x 4 with P straight from
//             registers (the S accumulator fragment is the A fragment of the next product, packed to fp16).
//   softmax   online over the chunks, rows in registers (quad shuffles), running max in the scaled log2 domain.
// The chunk order (all self keys, then all conditioning keys) differs from the mma.sync kernel's 64-key walk over the
// concatenated list only in the fp32 rounding of the online rescaling.
#include <cstdlib>

#include "attention.cuh"
#include "gemm.cuh"

namespace pb {

constexpr int AW_HD = 80;
constexpr int AW_BM = 64;                       // queries per CTA
constexpr int AW_BN = 64;                       // keys per chunk
constexpr int AW_K64 = AW_BN * 128;             // K dims 0..63, SWIZZLE_128B
constexpr int AW_K16 = AW_BN * 32;              // K dims 64..79, SWIZZLE_32B
constexpr int AW_VRAW = AW_BN * AW_HD * 2;      // V as loaded: [64 keys][80 dims]
constexpr int AW_STAGE = AW_K64 + AW_K16 + AW_VRAW;      // 20480 (multiple of 1024)
constexpr int AW_OFF_Q16 = AW_BM * 128;
constexpr int AW_OFF_STAGE = AW_OFF_Q16 + AW_BM * 32;    // 10240
constexpr int AW_OFF_VT = AW_OFF_STAGE + 2 * AW_STAGE;   // [80 dims][64 keys], SWIZZLE_128B
constexpr int AW_OFF_BAR = AW_OFF_VT + AW_HD * 128;
constexpr int AW_SMEM = AW_OFF_BAR + 64 + 1024;          // + alignment slack
constexpr int AW_OFF_SEGS = AW_OFF_BAR + 64;             // regional instance: the tile's AttnSegs
constexpr int AW_SMEM_REG = AW_OFF_SEGS + 256 + 1024;
static_assert(sizeof(AttnSegs) <= 256, "AttnSegs outgrew its shared-memory slot");

struct AttnMaps {
    CUtensorMap q64, q16, qv;      // over qkv [B*P, 3E]: 64x64 SW128, 16x64 SW32, 80x64 unswizzled boxes
    CUtensorMap c64, c16, cv;      // the same over ckv [slots*S_max, 2E]
};

// REG (attention_wgmma_kernel_regional): regional prompts (AttnRegion).  The tile walks its self keys, then the chunks of every
// prompt some query of it sees (attn_build_segs), each from the prompt's own first row; a row's keys of a prompt it does not
// see are masked the way keys at or past `valid` are, so its softmax is exact over the keys it sees.
// MAPS (attention_wgmma_kernel_maps, and with REG attention_wgmma_kernel_regional_maps): attention maps (AttnMapOut).  A map row
// also stores the scaled scores of its own conditioning's chunks (prompt 0's) and, at the end, its rows' log2-sum-exp; O takes the
// same arithmetic as the instance without maps.
// INJ (the _inject instances): prompt-to-prompt injection (AttnInject).  Q and the K boxes of every stage come from the source
// sample's row (self keys) or slot (its prompt 0's conditioning keys), the V box from the sample's own; the bytes of a stage are
// the same, so expect_tx is too.
// PERTURB (the _perturb instances): perturbed-attention guidance (AttnPerturb).  A perturbed sample's self chunks add their
// weighted P to a per-thread running self mass (rescaled like l_run, reduced over the quad at the end) and enter P V as zeros;
// the store adds mass * V_self of the query's own row before the division.
template <bool REG, bool MAPS, bool INJ, bool PERTURB = false>
__device__ __forceinline__ void attention_wgmma_body(const AttnMaps& maps, const AttnParams& p, const AttnRegion& rg,
                                                     const AttnMapOut& mo, const AttnInject& inj,
                                                     const AttnPerturb& pt = AttnPerturb{}) {
    pdl_launch_dependents();
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* gbase = smem_raw + (base - smem_u32(smem_raw));
    const uint32_t q_bar = base + AW_OFF_BAR;
    auto full_bar = [&](int s) { return base + AW_OFF_BAR + 8u + 8u * s; };

    const int tid = threadIdx.x, wq = tid >> 5, lane = tid & 31;
    const int q0 = blockIdx.x * AW_BM, h = blockIdx.y, b = blockIdx.z;
    const int E = p.E;
    const int n_self = p.self_attn ? p.P : 0;
    const int slot = p.kv_slot ? p.kv_slot[b] : b;
    const int n_cond = p.kv_len ? p.kv_len[slot] : p.S_max;
    const int Nk = n_self + n_cond;
    const int n_sc = (n_self + AW_BN - 1) / AW_BN;
    const int mr = MAPS ? attn_map_row(mo, b) : -1;
    const int qb = INJ ? attn_inj_src(inj, b) : b;                           // the sample whose Q and K this one uses
    const int kslot = INJ ? (p.kv_slot ? p.kv_slot[qb] : qb) : slot;
    const bool pert = PERTURB && attn_perturbed(pt, b);                       // CTA-uniform
    int n_chunks = n_sc + (n_cond + AW_BN - 1) / AW_BN;
    AttnSegs* segs = reinterpret_cast<AttnSegs*>(gbase + AW_OFF_SEGS);
    auto seg_of = [&](int c) {
        int si = 0;
        while (c >= segs->first[si + 1]) ++si;
        return si;
    };

    auto issue_chunk = [&](int c) {         // one thread
        const int st = c & 1;
        const uint32_t sb = base + AW_OFF_STAGE + st * AW_STAGE;
        ptx::mbar_arrive_expect_tx(full_bar(st), AW_STAGE);
        if constexpr (REG) {
            const int si = seg_of(c), k0 = (c - segs->first[si]) * AW_BN;
            if (segs->slot[si] < 0) {
                const int row = b * p.P + k0, krow = INJ ? qb * p.P + k0 : row;
                ptx::tma_load_2d(&maps.q64, full_bar(st), sb, E + h * AW_HD, krow);
                ptx::tma_load_2d(&maps.q16, full_bar(st), sb + AW_K64, E + h * AW_HD + 64, krow);
                ptx::tma_load_2d(&maps.qv, full_bar(st), sb + AW_K64 + AW_K16, 2 * E + h * AW_HD, row);
            } else {
                const int row = segs->slot[si] * p.S_max + k0;
                const int krow = INJ && segs->bit[si] == 0 ? kslot * p.S_max + k0 : row;
                ptx::tma_load_2d(&maps.c64, full_bar(st), sb, h * AW_HD, krow);
                ptx::tma_load_2d(&maps.c16, full_bar(st), sb + AW_K64, h * AW_HD + 64, krow);
                ptx::tma_load_2d(&maps.cv, full_bar(st), sb + AW_K64 + AW_K16, E + h * AW_HD, row);
            }
        } else if (c < n_sc) {
            const int row = b * p.P + c * AW_BN, krow = INJ ? qb * p.P + c * AW_BN : row;
            ptx::tma_load_2d(&maps.q64, full_bar(st), sb, E + h * AW_HD, krow);
            ptx::tma_load_2d(&maps.q16, full_bar(st), sb + AW_K64, E + h * AW_HD + 64, krow);
            ptx::tma_load_2d(&maps.qv, full_bar(st), sb + AW_K64 + AW_K16, 2 * E + h * AW_HD, row);
        } else {
            const int row = slot * p.S_max + (c - n_sc) * AW_BN, krow = INJ ? kslot * p.S_max + (c - n_sc) * AW_BN : row;
            ptx::tma_load_2d(&maps.c64, full_bar(st), sb, h * AW_HD, krow);
            ptx::tma_load_2d(&maps.c16, full_bar(st), sb + AW_K64, h * AW_HD + 64, krow);
            ptx::tma_load_2d(&maps.cv, full_bar(st), sb + AW_K64 + AW_K16, E + h * AW_HD, row);
        }
    };
    if constexpr (REG) {
        if (wq == 0) {
            const uint32_t u = attn_tile_union(p, rg, b, q0, lane);
            if (lane == 0) attn_build_segs(p, rg, b, u, false, *segs);
            __syncwarp();
            n_chunks = segs->first[segs->n];
        }
    }
    if (wq == 0 && ptx::elect_one()) {
        ptx::mbar_init(q_bar, 1);
        ptx::mbar_init(full_bar(0), 1);
        ptx::mbar_init(full_bar(1), 1);
        ptx::fence_barrier_init();
        ptx::mbar_arrive_expect_tx(q_bar, AW_BM * 160);
        ptx::tma_load_2d(&maps.q64, q_bar, base, h * AW_HD, qb * p.P + q0);
        ptx::tma_load_2d(&maps.q16, q_bar, base + AW_OFF_Q16, h * AW_HD + 64, qb * p.P + q0);
        for (int c = 0; c < 2 && c < n_chunks; ++c) issue_chunk(c);
    }
    __syncthreads();
    uint32_t row_mask[2] = {0u, 0u};
    if constexpr (REG) {
        n_chunks = segs->first[segs->n];
        for (int r = 0; r < 2; ++r) row_mask[r] = attn_row_mask(p, rg, b, q0 + wq * 16 + (lane >> 2) + 8 * r);
    }

    const float* w_row = nullptr;
    const int n_w = attn_weight_row(p, b, w_row);
    const bool weighted = n_w > 0;
    const int w_start = Nk - n_w;
    float o[AW_HD / 2];
#pragma unroll
    for (int i = 0; i < AW_HD / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-1e30f, -1e30f}, l_run[2] = {0.f, 0.f};
    float mass[2] = {0.f, 0.f};             // PERTURB: this thread's share of the running self mass
    const uint64_t dq64 = ptx::wgmma_desc_kmajor_sw128(base);      // the warpgroup's 64 rows are the whole query tile
    const uint64_t dq16 = ptx::wgmma_desc_kmajor_sw32(base + AW_OFF_Q16);
    ptx::mbar_wait(q_bar, 0);

    for (int c = 0; c < n_chunks; ++c) {
        const int st = c & 1;
        int k0, valid, key0, lim[2];
        bool own_cond;                      // a chunk of the sample's own conditioning keys (the map's keys)
        bool self_chunk;
        if constexpr (REG) {
            const int si = seg_of(c), bit = segs->bit[si];
            own_cond = bit == 0;
            self_chunk = bit < 0;
            k0 = (c - segs->first[si]) * AW_BN;
            valid = min(AW_BN, segs->len[si] - k0);
            key0 = bit < 0 ? k0 : bit == 0 ? n_self + k0 : Nk;              // only [self ; prompt 0] is weighted
            for (int r = 0; r < 2; ++r) lim[r] = (bit < 0 || ((row_mask[r] >> bit) & 1u)) ? valid : 0;
        } else {
            const bool self = c < n_sc;
            own_cond = !self;
            self_chunk = self;
            k0 = self ? c * AW_BN : (c - n_sc) * AW_BN;                      // first key of the chunk inside its source
            valid = min(AW_BN, (self ? n_self : n_cond) - k0);
            key0 = self ? k0 : n_self + k0;                                   // index in [self ; cond]
        }
        // keys at or past lim(i) are masked for the row of accumulator element i
        auto lim_of = [&](int i) {
            if constexpr (REG) return lim[(i >> 1) & 1];
            else return valid;
        };
        const uint32_t sb = base + AW_OFF_STAGE + st * AW_STAGE;
        ptx::mbar_wait(full_bar(st), (c >> 1) & 1);
        // V [key][dim] -> Vt [dim][key] with the 128-byte swizzle: the 80 8x8 blocks (8 key blocks x 10 dim blocks) through
        // ldmatrix.trans, 20 per warp; thread t receives dim 8 db + t/4, keys 8 kb + 2 (t%4) + {0, 1} = one 4-byte store.
        // Keys at or past `valid` are written as zeros: the 64-row box runs into the next sample's rows, or the slot's rows
        // past kv_len and the next slot, and their P of 0 would still turn an Inf or NaN there into NaN in O += P V.
        {
            const uint32_t vraw = sb + AW_K64 + AW_K16;
            uint8_t* vt = gbase + AW_OFF_VT;
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                const int ml = wq * 20 + j * 4 + (lane >> 3);          // the block whose row this lane addresses
                uint32_t r[4];
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                             : "r"(vraw + (uint32_t)(((ml & 7) * 8 + (lane & 7)) * (AW_HD * 2) + (ml >> 3) * 16)));
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int m = wq * 20 + j * 4 + q, kb = m & 7, d = (m >> 3) * 8 + (lane >> 2);
                    const int key = kb * 8 + 2 * (lane & 3), byte = 2 * key;
                    const uint32_t v2 = key + 1 < valid ? r[q] : key < valid ? r[q] & 0xffffu : 0u;
                    *reinterpret_cast<uint32_t*>(vt + d * 128 + (((byte >> 4) ^ (d & 7)) << 4) + (byte & 15)) = v2;
                }
            }
        }
        ptx::fence_proxy_async_smem();      // the transposed tile must be visible to the tensor core's async proxy
        __syncthreads();

        // ---- S = Q K^T
        float s[AW_BN / 2];
        ptx::wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
            ptx::wgmma_m64n64k16(s, dq64 + 2 * ks, ptx::wgmma_desc_kmajor_sw128(sb) + 2 * ks, ks != 0 ? 1u : 0u);
        ptx::wgmma_m64n64k16(s, dq16, ptx::wgmma_desc_kmajor_sw32(sb + AW_K64), 1u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(s);
        if constexpr (MAPS) {
            if (mr >= 0 && own_cond) {       // the conditioning keys k0 + col of rows lane/4 and lane/4 + 8 of the warp's 16
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int row = q0 + wq * 16 + (lane >> 2) + 8 * r;
                    if (row >= p.P) continue;
                    float* dst = mo.scores + (((int64_t)mr * p.nhead + h) * p.P + row) * p.S_max + k0;
#pragma unroll
                    for (int i = 0; i < AW_BN / 2; ++i) {
                        const int col = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
                        if (((i >> 1) & 1) == r && col < valid) dst[col] = s[i] * p.scale_log2;
                    }
                }
            }
        }

        // ---- mask, online softmax (rows lane/4 and lane/4 + 8 of the warp's 16; key column 8n + 2(lane%4) + i%2)
        float mx[2] = {-1e30f, -1e30f};
#pragma unroll
        for (int i = 0; i < AW_BN / 2; ++i) {
            const int col = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
            if (col >= lim_of(i)) s[i] = -1e30f;
            mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
        }
        float corr[2], rs[2] = {0.f, 0.f}, msc[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r] * p.scale_log2);     // scale > 0: max commutes with it
            corr[r] = exp2f(m_run[r] - m_new);
            m_run[r] = m_new;
            msc[r] = -m_new;
        }
#pragma unroll
        for (int i = 0; i < AW_BN / 2; ++i) {
            const int col = (i >> 2) * 8 + 2 * (lane & 3) + (i & 1);
            float pv = col < lim_of(i) ? exp2f(fmaf(s[i], p.scale_log2, msc[(i >> 1) & 1])) : 0.f;
            rs[(i >> 1) & 1] += pv;
            if (weighted) {       // post-softmax, un-renormalised scaling of the last n_w keys
                const int kj = key0 + col;
                if (kj >= w_start && col < lim_of(i) && (!REG || kj < Nk)) pv *= w_row[kj - w_start];
            }
            s[i] = pv;
        }
        if constexpr (PERTURB) {
            if (pert) {
                mass[0] *= corr[0];
                mass[1] *= corr[1];
                if (self_chunk) {
#pragma unroll
                    for (int i = 0; i < AW_BN / 2; ++i) {
                        mass[(i >> 1) & 1] += s[i];
                        s[i] = 0.f;
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
            rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
            l_run[r] = l_run[r] * corr[r] + rs[r];
        }
#pragma unroll
        for (int i = 0; i < AW_HD / 2; ++i) o[i] *= corr[(i >> 1) & 1];

        // ---- O += P V, P from registers
        ptx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < AW_BN / 16; ++kk) {
            const uint32_t a[4] = {pack_half2(s[8 * kk + 0], s[8 * kk + 1]), pack_half2(s[8 * kk + 2], s[8 * kk + 3]),
                                   pack_half2(s[8 * kk + 4], s[8 * kk + 5]), pack_half2(s[8 * kk + 6], s[8 * kk + 7])};
            ptx::wgmma_m64n80k16_rs(o, a, ptx::wgmma_desc_kmajor_sw128(base + AW_OFF_VT) + 2 * kk);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(o);
        __syncthreads();                    // stage st and Vt are free
        if (c + 2 < n_chunks && wq == 0 && ptx::elect_one()) issue_chunk(c + 2);
    }

    // ---- normalise and store
    if constexpr (PERTURB) {
        if (pert) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                mass[r] += __shfl_xor_sync(0xffffffffu, mass[r], 1);
                mass[r] += __shfl_xor_sync(0xffffffffu, mass[r], 2);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = q0 + wq * 16 + (lane >> 2) + 8 * r;
        if (row < p.P) {
            const float inv = 1.0f / l_run[r];
            __half* dst = p.out + ((int64_t)b * p.P + row) * E + h * AW_HD + 2 * (lane & 3);
            if constexpr (PERTURB) {
                if (pert) {         // the diagonal: mass * V_self of the query's own row
                    const __half* v = p.qkv + ((int64_t)b * p.P + row) * 3 * E + 2 * E + h * AW_HD + 2 * (lane & 3);
#pragma unroll
                    for (int n = 0; n < AW_HD / 8; ++n) {
                        const float2 vf = __half22float2(*reinterpret_cast<const __half2*>(v + n * 8));
                        o[4 * n + 2 * r] = fmaf(mass[r], vf.x, o[4 * n + 2 * r]);
                        o[4 * n + 2 * r + 1] = fmaf(mass[r], vf.y, o[4 * n + 2 * r + 1]);
                    }
                }
            }
#pragma unroll
            for (int n = 0; n < AW_HD / 8; ++n)
                *reinterpret_cast<uint32_t*>(dst + n * 8) = pack_half2(o[4 * n + 2 * r] * inv, o[4 * n + 2 * r + 1] * inv);
            if constexpr (MAPS)
                if (mr >= 0 && (lane & 3) == 0) mo.lse2[((int64_t)mr * p.nhead + h) * p.P + row] = m_run[r] + log2f(l_run[r]);
        }
    }
}

__global__ void __launch_bounds__(128) attention_wgmma_kernel(const __grid_constant__ AttnMaps maps, const AttnParams p) {
    attention_wgmma_body<false, false, false>(maps, p, AttnRegion{}, AttnMapOut{}, AttnInject{});
}
__global__ void __launch_bounds__(128) attention_wgmma_kernel_regional(const __grid_constant__ AttnMaps maps, const AttnParams p,
                                                                       const AttnRegion rg) {
    attention_wgmma_body<true, false, false>(maps, p, rg, AttnMapOut{}, AttnInject{});
}
__global__ void __launch_bounds__(128) attention_wgmma_kernel_maps(const __grid_constant__ AttnMaps maps, const AttnParams p,
                                                                   const AttnMapOut mo) {
    attention_wgmma_body<false, true, false>(maps, p, AttnRegion{}, mo, AttnInject{});
}
__global__ void __launch_bounds__(128) attention_wgmma_kernel_regional_maps(const __grid_constant__ AttnMaps maps, const AttnParams p,
                                                                            const AttnRegion rg, const AttnMapOut mo) {
    attention_wgmma_body<true, true, false>(maps, p, rg, mo, AttnInject{});
}
__global__ void __launch_bounds__(128) attention_wgmma_kernel_inject(const __grid_constant__ AttnMaps maps, const AttnParams p,
                                                                     const AttnInject inj) {
    attention_wgmma_body<false, false, true>(maps, p, AttnRegion{}, AttnMapOut{}, inj);
}
__global__ void __launch_bounds__(128) attention_wgmma_kernel_regional_inject(const __grid_constant__ AttnMaps maps, const AttnParams p,
                                                                              const AttnRegion rg, const AttnInject inj) {
    attention_wgmma_body<true, false, true>(maps, p, rg, AttnMapOut{}, inj);
}
__global__ void __launch_bounds__(128) attention_wgmma_kernel_maps_inject(const __grid_constant__ AttnMaps maps, const AttnParams p,
                                                                          const AttnMapOut mo, const AttnInject inj) {
    attention_wgmma_body<false, true, true>(maps, p, AttnRegion{}, mo, inj);
}
__global__ void __launch_bounds__(128) attention_wgmma_kernel_regional_maps_inject(const __grid_constant__ AttnMaps maps,
                                                                                   const AttnParams p, const AttnRegion rg,
                                                                                   const AttnMapOut mo, const AttnInject inj) {
    attention_wgmma_body<true, true, true>(maps, p, rg, mo, inj);
}

// every combination of the other flags, for the rows of the launch that are not perturbed
template <bool REG, bool MAPS, bool INJ>
__global__ void __launch_bounds__(128) attention_wgmma_kernel_perturb(const __grid_constant__ AttnMaps maps, const AttnParams p,
                                                                      const AttnRegion rg, const AttnMapOut mo, const AttnInject inj,
                                                                      const AttnPerturb pt) {
    attention_wgmma_body<REG, MAPS, INJ, true>(maps, p, rg, mo, inj, pt);
}

template <bool REG, bool MAPS, bool INJ>
static int launch_wgmma_perturb(dim3 grid, cudaStream_t st, const AttnMaps& m, const AttnParams& p, const AttnRegion* rg,
                                const AttnMapOut* mo, const AttnInject* inj, const AttnPerturb& pt) {
    constexpr int smem = REG ? AW_SMEM_REG : AW_SMEM;
    static DeviceOnce attr_once;
    if (attr_once.first())
        PB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel_perturb<REG, MAPS, INJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attention_wgmma_kernel_perturb<REG, MAPS, INJ><<<grid, 128, smem, st>>>(m, p, rg ? *rg : AttnRegion{}, mo ? *mo : AttnMapOut{},
                                                                             inj ? *inj : AttnInject{}, pt);
    return 0;
}

// returns 0 = launched, 1 = error, -1 = shape not handled here (head_dim != 80: the caller runs the mma.sync kernel)
int launch_attention_wgmma(const AttnParams& p, cudaStream_t st, const AttnRegion* rg, const AttnMapOut* mo, const AttnInject* inj,
                           const AttnPerturb* pt) {
    static const bool off = getenv("PB200_ATTN_MMA_SYNC") != nullptr;      // A/B knob: the mma.sync kernel for every shape
    if (off || p.E != AW_HD * p.nhead) return -1;
    const int64_t q_rows = (int64_t)p.B * p.P;
    const int64_t c_rows = (int64_t)(p.n_slots > 0 ? p.n_slots : p.B) * p.S_max;
    AttnMaps m;
    PB_TRY(cached_tmap_f16_2d(p.qkv, q_rows, 3 * (int64_t)p.E, 3 * (int64_t)p.E, 64, AW_BM, 128, &m.q64));
    PB_TRY(cached_tmap_f16_2d(p.qkv, q_rows, 3 * (int64_t)p.E, 3 * (int64_t)p.E, 16, AW_BM, 32, &m.q16));
    PB_TRY(cached_tmap_f16_2d(p.qkv, q_rows, 3 * (int64_t)p.E, 3 * (int64_t)p.E, AW_HD, AW_BN, 0, &m.qv));
    if (c_rows > 0) {
        PB_TRY(cached_tmap_f16_2d(p.ckv, c_rows, 2 * (int64_t)p.E, 2 * (int64_t)p.E, 64, AW_BN, 128, &m.c64));
        PB_TRY(cached_tmap_f16_2d(p.ckv, c_rows, 2 * (int64_t)p.E, 2 * (int64_t)p.E, 16, AW_BN, 32, &m.c16));
        PB_TRY(cached_tmap_f16_2d(p.ckv, c_rows, 2 * (int64_t)p.E, 2 * (int64_t)p.E, AW_HD, AW_BN, 0, &m.cv));
    } else {
        m.c64 = m.q64; m.c16 = m.q16; m.cv = m.qv;      // never read: no conditioning keys
    }
    ProfScope prof("attention", 2.0 * ((double)p.B * p.P * 4.0 * p.E + (double)p.B * p.S_max * 2.0 * p.E), st);
    dim3 grid(ceil_div(p.P, AW_BM), p.nhead, p.B);
    PB_CHECK(grid.y <= 65535 && grid.z <= 65535, "attention: grid too large");
#define PB_AW_LAUNCH(KERNEL, SMEM, ...)                                                                 \
    {                                                                                                   \
        static DeviceOnce attr_once;                                                                    \
        if (attr_once.first()) PB_CUDA(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM)); \
        KERNEL<<<grid, 128, SMEM, st>>>(m, p, __VA_ARGS__);                                             \
    }
    if (pt != nullptr) {
        const bool r = rg != nullptr, mp = mo != nullptr, in = inj != nullptr;
        if (r && mp && in) PB_TRY((launch_wgmma_perturb<true, true, true>(grid, st, m, p, rg, mo, inj, *pt)));
        else if (r && mp) PB_TRY((launch_wgmma_perturb<true, true, false>(grid, st, m, p, rg, mo, inj, *pt)));
        else if (r && in) PB_TRY((launch_wgmma_perturb<true, false, true>(grid, st, m, p, rg, mo, inj, *pt)));
        else if (mp && in) PB_TRY((launch_wgmma_perturb<false, true, true>(grid, st, m, p, rg, mo, inj, *pt)));
        else if (r) PB_TRY((launch_wgmma_perturb<true, false, false>(grid, st, m, p, rg, mo, inj, *pt)));
        else if (mp) PB_TRY((launch_wgmma_perturb<false, true, false>(grid, st, m, p, rg, mo, inj, *pt)));
        else if (in) PB_TRY((launch_wgmma_perturb<false, false, true>(grid, st, m, p, rg, mo, inj, *pt)));
        else PB_TRY((launch_wgmma_perturb<false, false, false>(grid, st, m, p, rg, mo, inj, *pt)));
    } else if (inj != nullptr) {
        if (mo != nullptr && rg != nullptr) PB_AW_LAUNCH(attention_wgmma_kernel_regional_maps_inject, AW_SMEM_REG, *rg, *mo, *inj)
        else if (mo != nullptr) PB_AW_LAUNCH(attention_wgmma_kernel_maps_inject, AW_SMEM, *mo, *inj)
        else if (rg != nullptr) PB_AW_LAUNCH(attention_wgmma_kernel_regional_inject, AW_SMEM_REG, *rg, *inj)
        else PB_AW_LAUNCH(attention_wgmma_kernel_inject, AW_SMEM, *inj)
    } else if (mo != nullptr && rg != nullptr) {
        static DeviceOnce attr_reg_maps;
        if (attr_reg_maps.first())
            PB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel_regional_maps, cudaFuncAttributeMaxDynamicSharedMemorySize, AW_SMEM_REG));
        attention_wgmma_kernel_regional_maps<<<grid, 128, AW_SMEM_REG, st>>>(m, p, *rg, *mo);
    } else if (mo != nullptr) {
        static DeviceOnce attr_maps;
        if (attr_maps.first())
            PB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel_maps, cudaFuncAttributeMaxDynamicSharedMemorySize, AW_SMEM));
        attention_wgmma_kernel_maps<<<grid, 128, AW_SMEM, st>>>(m, p, *mo);
    } else if (rg != nullptr) {
        static DeviceOnce attr_reg;
        if (attr_reg.first())
            PB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel_regional, cudaFuncAttributeMaxDynamicSharedMemorySize, AW_SMEM_REG));
        attention_wgmma_kernel_regional<<<grid, 128, AW_SMEM_REG, st>>>(m, p, *rg);
    } else {
        static DeviceOnce attr;
        if (attr.first())
            PB_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AW_SMEM));
        attention_wgmma_kernel<<<grid, 128, AW_SMEM, st>>>(m, p);
    }
#undef PB_AW_LAUNCH
    PB_LAUNCH_CHECK();
    return 0;
}

}  // namespace pb
