// Attention core of AttnBlock: softmax(q k^T / sqrt(hd)) v over keys = [self tokens ; conditioning tokens].
// Replaces nn.MultiheadAttention's SDPA (ref/src/modules.py:10,17) and the explicit matmul/softmax/matmul of
// CustomMultiheadAttention incl. its post-softmax `attn_weights` (ref/utils/alter_attention.py:19-36).
//
// At the reference's shapes this op is HBM/latency bound, not tensor bound: <=256 queries x <=1032 keys x 16
// heads x hd 80 per sample is ~1% of a forward's FLOPs (SURVEY.md §8a R7), and one (sample, head) problem is far
// smaller than a 128-row GEMM tile.  So: one CTA per (64 queries, head, sample), flash-style online softmax over
// 64-key chunks.  head_dim 80 runs the wgmma + TMA kernel of attention_wg.cu; this file's kernel (fp16 mma.sync
// m16n8k16 with fp32 accumulation, K/V staged in padded shared memory and read with ldmatrix) every other head dim.
// The projections around it (QKV, out_proj) are the wgmma GEMMs in gemm.cu.
#include "attention.cuh"

namespace pb {

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 16-byte asynchronous global->shared copy; src_bytes = 0 zero-fills the destination
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

constexpr int ATT_BM = 64;   // queries per CTA (4 warps x 16)
constexpr int ATT_BN = 64;   // keys per chunk
constexpr float NEG_BIG = -1e30f;

// One CTA per (64 queries, head, sample); each warp owns 16 queries and walks the keys in 64-key chunks
// (double-buffered cp.async).  It runs every head dim other than 80 (csrc/attention_wg.cu), and head_dim 80 with
// PB200_ATTN_MMA_SYNC=1.  REG (attention_kernel_regional): regional prompts (AttnRegion): the tile walks [self ; prompt 0]
// as above, then the chunks of every further prompt some query of it sees, each from the prompt's own first row
// (attn_build_segs); a row's keys of a prompt it does not see are masked like keys past the end, so its softmax is exact over
// the keys it sees.  MAPS (attention_kernel_maps, and with REG attention_kernel_regional_maps): attention maps (AttnMapOut); a map
// row also stores the scaled scores of its own conditioning keys (prompt 0's) and, at the end, its rows' log2-sum-exp, and O takes
// the same arithmetic as the instance without maps.  INJ (the _inject instances): prompt-to-prompt injection (AttnInject); Q and
// the K rows come from the source sample's row (self keys) or slot (its prompt 0's conditioning keys), the V rows from the
// sample's own, so ks and vs have separate bases.  PERTURB (the _perturb instances): perturbed-attention guidance (AttnPerturb); a
// perturbed sample's self keys (those before the chunk walk's first conditioning key) add their weighted P to a per-thread running
// self mass and enter P V as zeros, and the store adds mass * V_self of the query's own row before the division.
template <int HD, bool REG, bool MAPS, bool INJ, bool PERTURB = false>
__device__ __forceinline__ void attention_body(const AttnParams& p, const AttnRegion& rg, const AttnMapOut& mo, const AttnInject& inj,
                                               const AttnPerturb& pt = AttnPerturb{}) {
    constexpr int LDS = HD + 8;           // padded row: (HD+8)*2 bytes is an odd multiple of 16 -> conflict-free ldmatrix
    constexpr int CPR = HD / 8;           // 16-byte chunks per row
    constexpr int QROWS = ATT_BM;
    constexpr int n_buf = 2;
    pdl_launch_dependents();
    extern __shared__ __align__(16) __half smem_att[];
    __half* sQ = smem_att;                                   // [QROWS][LDS]
    __half* sKb = smem_att + QROWS * LDS;                     // [n_buf][ATT_BN][LDS]
    __half* sVb = sKb + n_buf * ATT_BN * LDS;                 // [n_buf][ATT_BN][LDS]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int q0 = blockIdx.x * QROWS, h = blockIdx.y, b = blockIdx.z;
    const int E = p.E;
    const int64_t ldq = 3 * (int64_t)E, ldc = 2 * (int64_t)E;
    const int n_self = p.self_attn ? p.P : 0;
    const int slot = p.kv_slot ? p.kv_slot[b] : b;            // samples with identical conditioning share one K/V block
    const int n_cond = p.kv_len ? p.kv_len[slot] : p.S_max;
    const int Nk = n_self + n_cond;
    const int mr = MAPS ? attn_map_row(mo, b) : -1;
    const bool pert = PERTURB && attn_perturbed(pt, b);        // CTA-uniform
    const __half* qkv_b = p.qkv + (int64_t)b * p.P * ldq;
    const __half* ckv_b = p.ckv + (int64_t)slot * p.S_max * ldc;
    const int qb = INJ ? attn_inj_src(inj, b) : b;            // the sample whose Q and K this one uses
    const __half* qkv_k = INJ ? p.qkv + (int64_t)qb * p.P * ldq : qkv_b;
    const __half* ckv_k = INJ ? p.ckv + (int64_t)(p.kv_slot ? p.kv_slot[qb] : qb) * p.S_max * ldc : ckv_b;
    AttnSegs* segs = reinterpret_cast<AttnSegs*>(sVb + n_buf * ATT_BN * LDS);
    if constexpr (REG) {
        if (warp == 0) {
            const uint32_t u = attn_tile_union(p, rg, b, q0, lane);
            if (lane == 0) attn_build_segs(p, rg, b, u, true, *segs);
        }
        __syncthreads();
    }

    // K/V chunk j0.. -> buffer `buf` with 16-byte cp.async (zero-fill for keys past the end)
    auto load_chunk = [&](int j0, int buf) {
        __half* sK = sKb + buf * ATT_BN * LDS;
        __half* sV = sVb + buf * ATT_BN * LDS;
        for (int c = tid; c < ATT_BN * CPR; c += 128) {
            const int r = c / CPR, cc = c - r * CPR;
            const int j = j0 + r;
            const __half *ks = qkv_b, *vs = qkv_b;
            uint32_t nbytes = 0;
            if (j < n_self) {
                ks = qkv_k + (int64_t)j * ldq + h * HD + cc * 8 + E;
                vs = INJ ? qkv_b + (int64_t)j * ldq + h * HD + cc * 8 + 2 * E : ks + E;
                nbytes = 16;
            } else if (j < Nk) {
                ks = ckv_k + (int64_t)(j - n_self) * ldc + h * HD + cc * 8;
                vs = INJ ? ckv_b + (int64_t)(j - n_self) * ldc + h * HD + cc * 8 + E : ks + E;
                nbytes = 16;
            }
            cp_async16(smem_u32(sK + r * LDS + cc * 8), ks, nbytes);
            cp_async16(smem_u32(sV + r * LDS + cc * 8), vs, nbytes);
        }
    };
    // chunk c of the regional walk -> buffer `buf`: keys before the segment's `from` are self keys, the rest its prompt's rows
    auto load_chunk_reg = [&](int c, int buf) {
        int si = 0;
        while (c >= segs->first[si + 1]) ++si;
        const int j0 = (c - segs->first[si]) * ATT_BN, len = segs->len[si], from = segs->from[si];
        const __half* cb = p.ckv + (int64_t)segs->slot[si] * p.S_max * ldc;
        const __half* cb_k = INJ && segs->bit[si] == 0 ? ckv_k : cb;
        __half* sK = sKb + buf * ATT_BN * LDS;
        __half* sV = sVb + buf * ATT_BN * LDS;
        for (int i = tid; i < ATT_BN * CPR; i += 128) {
            const int r = i / CPR, cc = i - r * CPR;
            const int j = j0 + r;
            const __half *ks = qkv_b, *vs = qkv_b;
            uint32_t nbytes = 0;
            if (j < from) {
                ks = qkv_k + (int64_t)j * ldq + h * HD + cc * 8 + E;
                vs = INJ ? qkv_b + (int64_t)j * ldq + h * HD + cc * 8 + 2 * E : ks + E;
                nbytes = 16;
            } else if (j < len) {
                ks = cb_k + (int64_t)(j - from) * ldc + h * HD + cc * 8;
                vs = INJ ? cb + (int64_t)(j - from) * ldc + h * HD + cc * 8 + E : ks + E;
                nbytes = 16;
            }
            cp_async16(smem_u32(sK + r * LDS + cc * 8), ks, nbytes);
            cp_async16(smem_u32(sV + r * LDS + cc * 8), vs, nbytes);
        }
    };
    // Q rides in the same cp.async group as the first K/V chunk (a register-staged Q load costs 5 serialised global
    // round trips before anything else can start)
    for (int c = tid; c < QROWS * CPR; c += 128) {
        const int r = c / CPR, cc = c - r * CPR;
        const bool ok = q0 + r < p.P;
        cp_async16(smem_u32(sQ + r * LDS + cc * 8), ok ? qkv_k + (int64_t)(q0 + r) * ldq + h * HD + cc * 8 : qkv_k, ok ? 16u : 0u);
    }
    int n_chunks = 0;
    if constexpr (REG) {
        n_chunks = segs->first[segs->n];
        if (n_chunks > 0) load_chunk_reg(0, 0);
    } else {
        load_chunk(0, 0);
    }
    cp_async_commit();

    const int qrow0 = warp * 16;                              // this warp's 16 query rows inside the tile
    uint32_t qf[HD / 16][4];
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_run[2] = {NEG_BIG, NEG_BIG}, l_run[2] = {0.f, 0.f};
    float mass[2] = {0.f, 0.f};                               // PERTURB: this thread's share of the running self mass

    const float* w_row = nullptr;
    const int n_w = attn_weight_row(p, b, w_row);
    const bool weighted = n_w > 0;
    const int w_start = Nk - n_w;
    uint32_t row_mask[2] = {0u, 0u};
    if constexpr (REG)
        for (int r = 0; r < 2; ++r) row_mask[r] = attn_row_mask(p, rg, b, q0 + warp * 16 + g + 8 * r);

    auto load_q_frags = [&]() {
#pragma unroll
        for (int ks = 0; ks < HD / 16; ++ks)
            ldmatrix_x4(qf[ks], smem_u32(sQ + (qrow0 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8));
    };

    // one online-softmax pass of this warp's 16 query rows over the 64 keys j0.. held in (sK, sV); regional: of a segment of
    // seg_nk keys, bit `bit` of a row's mask gating its keys from `from` on
    auto process_chunk = [&](int j0, const __half* sK, const __half* sV, int seg_nk, int from, int bit) {
        auto visible = [&](int key, int r) { return key < seg_nk && (key < from || ((row_mask[r] >> bit) & 1u)); };
        const bool full = !REG && j0 + ATT_BN <= Nk;      // warp-uniform: no key of this chunk is masked
        // ---- S = Q K^T
        float s[ATT_BN / 8][4];
#pragma unroll
        for (int i = 0; i < ATT_BN / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
        for (int np = 0; np < ATT_BN / 16; ++np) {
            if (j0 + np * 16 >= (REG ? seg_nk : Nk)) break;    // 16-key groups past the end are fully masked
#pragma unroll
            for (int ks = 0; ks < HD / 16; ++ks) {
                uint32_t kf[4];
                ldmatrix_x4(kf, smem_u32(sK + (np * 16 + (lane & 7) + ((lane >> 4) << 3)) * LDS + ks * 16 + ((lane >> 3) & 1) * 8));
                mma_16816(s[2 * np], qf[ks], kf[0], kf[1]);
                mma_16816(s[2 * np + 1], qf[ks], kf[2], kf[3]);
            }
        }
        if constexpr (MAPS) {
            // the chunk's own conditioning keys j - c_from: [n_self, Nk), or regional prompt 0's part of segment 0
            const int c_from = REG ? from : n_self, c_end = REG ? seg_nk : Nk;
            if (mr >= 0 && (!REG || bit == 0) && j0 + ATT_BN > c_from) {
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int row = q0 + warp * 16 + g + 8 * r;
                    if (row >= p.P) continue;
                    float* dst = mo.scores + (((int64_t)mr * p.nhead + h) * p.P + row) * p.S_max;
#pragma unroll
                    for (int nt = 0; nt < ATT_BN / 8; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int key = j0 + nt * 8 + 2 * t + e;
                            if (key >= c_from && key < c_end) dst[key - c_from] = s[nt][2 * r + e] * p.scale_log2;
                        }
                }
            }
        }
        // ---- mask, online softmax (rows g and g+8 of the warp's 16).  The running max is kept in the scaled log2
        // domain; the 1/sqrt(hd)*log2(e) factor is folded into the exp2 argument's FFMA.
        float mx[2] = {NEG_BIG, NEG_BIG};
        if (full) {
#pragma unroll
            for (int nt = 0; nt < ATT_BN / 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
        } else {
#pragma unroll
            for (int nt = 0; nt < ATT_BN / 8; ++nt) {
                const int key = j0 + nt * 8 + 2 * t;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if constexpr (REG) {
                        if (!visible(key + (e & 1), e >> 1)) s[nt][e] = NEG_BIG;
                    } else {
                        if (key + (e & 1) >= Nk) s[nt][e] = NEG_BIG;
                    }
                    mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
                }
            }
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
        for (int nt = 0; nt < ATT_BN / 8; ++nt) {
            if (!full && j0 + (nt >> 1) * 16 >= (REG ? seg_nk : Nk)) break;      // same groups the MMAs skip
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float pv = exp2f(fmaf(s[nt][e], p.scale_log2, msc[e >> 1]));
                // a row may see no key of this chunk yet: its running max is then the mask value itself
                if constexpr (REG) pv = visible(j0 + nt * 8 + 2 * t + (e & 1), e >> 1) ? pv : 0.f;
                rs[e >> 1] += pv;
                s[nt][e] = pv;
            }
        }
        if (weighted && (!REG || bit == 0)) {       // post-softmax, un-renormalised scaling of the last n_w key columns
#pragma unroll
            for (int nt = 0; nt < ATT_BN / 8; ++nt) {
                const int key = j0 + nt * 8 + 2 * t;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int kj = key + (e & 1);
                    if (kj >= w_start && kj < Nk) s[nt][e] *= w_row[kj - w_start];
                }
            }
        }
        if constexpr (PERTURB) {
            if (pert) {
                mass[0] *= corr[0];
                mass[1] *= corr[1];
                const int self_end = REG ? from : n_self;      // keys before it are self keys
                if (j0 < self_end) {
#pragma unroll
                    for (int nt = 0; nt < ATT_BN / 8; ++nt)
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            if (j0 + nt * 8 + 2 * t + (e & 1) < self_end) {
                                mass[e >> 1] += s[nt][e];
                                s[nt][e] = 0.f;
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
        for (int i = 0; i < HD / 8; ++i) {
            o[i][0] *= corr[0]; o[i][1] *= corr[0];
            o[i][2] *= corr[1]; o[i][3] *= corr[1];
        }
        // ---- O += P V
#pragma unroll
        for (int kk = 0; kk < ATT_BN / 16; ++kk) {
            if (j0 + kk * 16 >= (REG ? seg_nk : Nk)) break;    // P is zero there
            uint32_t a[4];
            a[0] = pack_half2(s[2 * kk][0], s[2 * kk][1]);
            a[1] = pack_half2(s[2 * kk][2], s[2 * kk][3]);
            a[2] = pack_half2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
            a[3] = pack_half2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
            for (int np = 0; np < HD / 16; ++np) {
                uint32_t vf[4];
                ldmatrix_x4_trans(vf, smem_u32(sV + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + np * 16 + (lane >> 4) * 8));
                mma_16816(o[2 * np], a, vf[0], vf[1]);
                mma_16816(o[2 * np + 1], a, vf[2], vf[3]);
            }
        }
    };

    const bool warp_active = q0 + warp * 16 < p.P;       // warps past the last query only help with the loads
    int buf = 0;
    if constexpr (REG) {
        for (int c = 0; c < n_chunks; ++c, buf ^= 1) {
            if (c + 1 < n_chunks) load_chunk_reg(c + 1, buf ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
            __syncthreads();
            if (c == 0) load_q_frags();
            if (warp_active) {
                int si = 0;
                while (c >= segs->first[si + 1]) ++si;
                process_chunk((c - segs->first[si]) * ATT_BN, sKb + buf * ATT_BN * LDS, sVb + buf * ATT_BN * LDS, segs->len[si],
                              segs->from[si], segs->bit[si]);
            }
            __syncthreads();
        }
    } else for (int j0 = 0; j0 < Nk; j0 += ATT_BN, buf ^= 1) {
        // prefetch the next chunk into the other buffer (all warps finished reading it at the end of the last iteration)
        if (j0 + ATT_BN < Nk) load_chunk(j0 + ATT_BN, buf ^ 1);
        cp_async_commit();
        cp_async_wait<1>();               // this chunk has landed (the prefetch may still be in flight)
        __syncthreads();
        if (j0 == 0) load_q_frags();
        if (warp_active) process_chunk(j0, sKb + buf * ATT_BN * LDS, sVb + buf * ATT_BN * LDS, 0, 0, 0);
        __syncthreads();                  // everyone is done with this buffer before it is refilled
    }
    cp_async_wait<0>();
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
        const int row = q0 + warp * 16 + g + r * 8;
        if (row < p.P) {
            const float inv = 1.0f / l_run[r];
            __half* dst = p.out + ((int64_t)b * p.P + row) * E + h * HD + 2 * t;
            if constexpr (PERTURB) {
                if (pert) {         // the diagonal: mass * V_self of the query's own row
                    const __half* v = qkv_b + (int64_t)row * ldq + 2 * E + h * HD + 2 * t;
#pragma unroll
                    for (int nt = 0; nt < HD / 8; ++nt) {
                        const float2 vf = __half22float2(*reinterpret_cast<const __half2*>(v + nt * 8));
                        o[nt][2 * r] = fmaf(mass[r], vf.x, o[nt][2 * r]);
                        o[nt][2 * r + 1] = fmaf(mass[r], vf.y, o[nt][2 * r + 1]);
                    }
                }
            }
#pragma unroll
            for (int nt = 0; nt < HD / 8; ++nt)
                *reinterpret_cast<uint32_t*>(dst + nt * 8) = pack_half2(o[nt][2 * r] * inv, o[nt][2 * r + 1] * inv);
            if constexpr (MAPS)
                if (mr >= 0 && t == 0) mo.lse2[((int64_t)mr * p.nhead + h) * p.P + row] = m_run[r] + log2f(l_run[r]);
        }
    }
}

template <int HD>
__global__ void __launch_bounds__(128) attention_kernel(const AttnParams p) {
    attention_body<HD, false, false, false>(p, AttnRegion{}, AttnMapOut{}, AttnInject{});
}
template <int HD>
__global__ void __launch_bounds__(128) attention_kernel_regional(const AttnParams p, const AttnRegion rg) {
    attention_body<HD, true, false, false>(p, rg, AttnMapOut{}, AttnInject{});
}
template <int HD>
__global__ void __launch_bounds__(128) attention_kernel_maps(const AttnParams p, const AttnMapOut mo) {
    attention_body<HD, false, true, false>(p, AttnRegion{}, mo, AttnInject{});
}
// (min blocks 1 on the regional maps and regional inject instances: at head_dim 80 the default register target spills)
template <int HD>
__global__ void __launch_bounds__(128, 1) attention_kernel_regional_maps(const AttnParams p, const AttnRegion rg, const AttnMapOut mo) {
    attention_body<HD, true, true, false>(p, rg, mo, AttnInject{});
}
template <int HD>
__global__ void __launch_bounds__(128) attention_kernel_inject(const AttnParams p, const AttnInject inj) {
    attention_body<HD, false, false, true>(p, AttnRegion{}, AttnMapOut{}, inj);
}
template <int HD>
__global__ void __launch_bounds__(128, 1) attention_kernel_regional_inject(const AttnParams p, const AttnRegion rg, const AttnInject inj) {
    attention_body<HD, true, false, true>(p, rg, AttnMapOut{}, inj);
}
template <int HD>
__global__ void __launch_bounds__(128) attention_kernel_maps_inject(const AttnParams p, const AttnMapOut mo, const AttnInject inj) {
    attention_body<HD, false, true, true>(p, AttnRegion{}, mo, inj);
}
template <int HD>
__global__ void __launch_bounds__(128, 1) attention_kernel_regional_maps_inject(const AttnParams p, const AttnRegion rg,
                                                                                const AttnMapOut mo, const AttnInject inj) {
    attention_body<HD, true, true, true>(p, rg, mo, inj);
}

// every combination of the other flags, for the rows of the launch that are not perturbed (min blocks 1 with regions, as above)
template <int HD, bool MAPS, bool INJ>
__global__ void __launch_bounds__(128) attention_kernel_perturb(const AttnParams p, const AttnMapOut mo, const AttnInject inj,
                                                                const AttnPerturb pt) {
    attention_body<HD, false, MAPS, INJ, true>(p, AttnRegion{}, mo, inj, pt);
}
template <int HD, bool MAPS, bool INJ>
__global__ void __launch_bounds__(128, 1) attention_kernel_regional_perturb(const AttnParams p, const AttnRegion rg, const AttnMapOut mo,
                                                                            const AttnInject inj, const AttnPerturb pt) {
    attention_body<HD, true, MAPS, INJ, true>(p, rg, mo, inj, pt);
}

template <int HD, bool REG, bool MAPS, bool INJ>
static int launch_perturb(dim3 grid, size_t smem, cudaStream_t st, const AttnParams& p, const AttnRegion* rg, const AttnMapOut* mo,
                          const AttnInject* inj, const AttnPerturb& pt) {
    static DeviceOnce attr_once;
    const AttnMapOut mo0 = mo ? *mo : AttnMapOut{};
    const AttnInject inj0 = inj ? *inj : AttnInject{};
    if constexpr (REG) {
        if (attr_once.first())
            PB_CUDA(cudaFuncSetAttribute(attention_kernel_regional_perturb<HD, MAPS, INJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attention_kernel_regional_perturb<HD, MAPS, INJ><<<grid, 128, smem, st>>>(p, *rg, mo0, inj0, pt);
    } else {
        if (attr_once.first())
            PB_CUDA(cudaFuncSetAttribute(attention_kernel_perturb<HD, MAPS, INJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attention_kernel_perturb<HD, MAPS, INJ><<<grid, 128, smem, st>>>(p, mo0, inj0, pt);
    }
    return 0;
}

template <int HD>
static int launch_perturb_hd(dim3 grid, size_t smem, cudaStream_t st, const AttnParams& p, const AttnRegion* rg, const AttnMapOut* mo,
                             const AttnInject* inj, const AttnPerturb& pt) {
    const bool r = rg != nullptr, mp = mo != nullptr, in = inj != nullptr;
    if (r && mp && in) return launch_perturb<HD, true, true, true>(grid, smem, st, p, rg, mo, inj, pt);
    if (r && mp) return launch_perturb<HD, true, true, false>(grid, smem, st, p, rg, mo, inj, pt);
    if (r && in) return launch_perturb<HD, true, false, true>(grid, smem, st, p, rg, mo, inj, pt);
    if (mp && in) return launch_perturb<HD, false, true, true>(grid, smem, st, p, rg, mo, inj, pt);
    if (r) return launch_perturb<HD, true, false, false>(grid, smem, st, p, rg, mo, inj, pt);
    if (mp) return launch_perturb<HD, false, true, false>(grid, smem, st, p, rg, mo, inj, pt);
    if (in) return launch_perturb<HD, false, false, true>(grid, smem, st, p, rg, mo, inj, pt);
    return launch_perturb<HD, false, false, false>(grid, smem, st, p, rg, mo, inj, pt);
}

int launch_attention(const AttnParams& p, cudaStream_t st, const AttnRegion* rg, const AttnMapOut* mo, const AttnInject* inj,
                     const AttnPerturb* pt) {
    PB_CHECK(p.nhead > 0 && p.E % p.nhead == 0, "attention: E=%d not divisible by nhead=%d", p.E, p.nhead);
    const int hd = p.E / p.nhead;
    PB_CHECK(p.E % 8 == 0, "attention: E must be a multiple of 8");
    if (p.B == 0 || p.P == 0) return 0;
    {
        const int rc = launch_attention_wgmma(p, st, rg, mo, inj, pt);
        if (rc >= 0) return rc;
    }
    // algorithmic bytes: q, self k/v, out once; conditioning k/v once per sample
    ProfScope prof("attention", 2.0 * ((double)p.B * p.P * 4.0 * p.E + (double)p.B * p.S_max * 2.0 * p.E), st);
    dim3 grid(ceil_div(p.P, ATT_BM), p.nhead, p.B);
    PB_CHECK(grid.y <= 65535 && grid.z <= 65535, "attention: grid too large");
    const bool reg = rg != nullptr;
    const size_t smem = (size_t)(ATT_BM + 4 * ATT_BN) * (hd + 8) * sizeof(__half) + (reg ? sizeof(AttnSegs) : 0);
#define PB_ATT_LAUNCH(KERNEL, ...)                                                                                  \
    {                                                                                                               \
        static DeviceOnce attr_once;                                                                                \
        if (attr_once.first()) PB_CUDA(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        KERNEL<<<grid, 128, smem, st>>>(p, __VA_ARGS__);                                                            \
        break;                                                                                                      \
    }
    switch (hd) {
#define PB_ATT_CASE(H)                                                                                              \
    case H: {                                                                                                       \
        if (pt != nullptr) {                                                                                        \
            PB_TRY(launch_perturb_hd<H>(grid, smem, st, p, rg, mo, inj, *pt));                                      \
            break;                                                                                                  \
        }                                                                                                           \
        if (inj != nullptr && mo != nullptr && reg) PB_ATT_LAUNCH(attention_kernel_regional_maps_inject<H>, *rg, *mo, *inj) \
        if (inj != nullptr && mo != nullptr) PB_ATT_LAUNCH(attention_kernel_maps_inject<H>, *mo, *inj)              \
        if (inj != nullptr && reg) PB_ATT_LAUNCH(attention_kernel_regional_inject<H>, *rg, *inj)                    \
        if (inj != nullptr) PB_ATT_LAUNCH(attention_kernel_inject<H>, *inj)                                         \
        if (mo != nullptr && reg) {                                                                                 \
            static DeviceOnce attr_reg_maps;                                                                        \
            if (attr_reg_maps.first())                                                                              \
                PB_CUDA(cudaFuncSetAttribute(attention_kernel_regional_maps<H>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            attention_kernel_regional_maps<H><<<grid, 128, smem, st>>>(p, *rg, *mo);                                \
            break;                                                                                                  \
        }                                                                                                           \
        if (mo != nullptr) {                                                                                        \
            static DeviceOnce attr_maps;                                                                            \
            if (attr_maps.first())                                                                                  \
                PB_CUDA(cudaFuncSetAttribute(attention_kernel_maps<H>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            attention_kernel_maps<H><<<grid, 128, smem, st>>>(p, *mo);                                              \
            break;                                                                                                  \
        }                                                                                                           \
        if (reg) {                                                                                                  \
            static DeviceOnce attr_reg;                                                                             \
            if (attr_reg.first())                                                                                   \
                PB_CUDA(cudaFuncSetAttribute(attention_kernel_regional<H>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            attention_kernel_regional<H><<<grid, 128, smem, st>>>(p, *rg);                                          \
            break;                                                                                                  \
        }                                                                                                           \
        static DeviceOnce attr;                                                                                   \
        if (attr.first()) {                                                                                                \
            PB_CUDA(cudaFuncSetAttribute(attention_kernel<H>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        }                                                                                                           \
        attention_kernel<H><<<grid, 128, smem, st>>>(p);                                                            \
        break;                                                                                                      \
    }
        PB_ATT_CASE(16) PB_ATT_CASE(32) PB_ATT_CASE(64) PB_ATT_CASE(80) PB_ATT_CASE(96)
#undef PB_ATT_CASE
#undef PB_ATT_LAUNCH
        default: PB_CHECK(false, "attention: head_dim %d unsupported (16/32/64/80/96)", hd);
    }
    PB_LAUNCH_CHECK();
    return 0;
}

}  // namespace pb
