// LoRA adapters per row: y += s * (alpha/r) * (x A^T) B^T after a linear layer's own GEMM, segmented by adapter.
//   Attention2D / nn.MultiheadAttention in_proj, out_proj   ref/src/modules.py:12-19
//   AttnBlock.kv_mapper                                     ref/src/modules.py:76-79
// A row with adapter a at scale s then equals the reference layer with W + s (alpha/r) B A.
//
// Two kernels over tiles of 32 rows, each running the distinct adapters among a tile's rows in ascending id order:
//   shrink  one CTA per tile; warp w owns ranks [w*RJ, (w+1)*RJ); lane l sums k in {8l + 256i .. +7} in ascending order, then a
//           fixed xor-butterfly over the 32 lanes; U = x A^T (fp32, [M][8 RJ]) goes to a scratch buffer.
//   expand  one CTA per (tile, 512 output columns); thread t owns columns n, n + 1 (n = 2t) and holds B[n, :], B[n + 1, :] in
//           registers; U rows are read from shared memory by broadcast, the sum over j runs in ascending order (zero-padded
//           ranks add exact zeros at the end), and the y pairs of eight rows are loaded together before they are updated.
// They are separate launches so that the expand -- which carries all the y traffic -- spreads over N as well as M (a fused kernel
// runs one CTA per 32 rows, too few for the AttnBlocks of the deepest level), without recomputing the shrink per column chunk.
// A row's result does not depend on the other rows of its tile, their adapters or RJ.  Rows with id -1 (or scale 0) take no
// part: their x, U and y rows are never touched.
#include <climits>

#include "lora.cuh"

namespace pb {

constexpr int LORA_TM = 32;
constexpr int LORA_THREADS = 256;
constexpr int LORA_WARPS = LORA_THREADS / 32;
constexpr int LORA_NCHUNK = 2 * LORA_THREADS;     // expand: output columns per CTA

struct LoraArgs {
    const __half* x;
    int64_t ldx, M;
    int K, N, rpe;
    const int* row_adapter;
    const float* row_scale;
    const int64_t* ln_stat;
    float* u;               // [M][RMAX] the shrink's output
    void* y;
    int64_t ldy;
    int remap_in, remap_out;
};

__device__ __forceinline__ void unpack8(const uint4 v, float (&f)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}

// ---- shrink: u[m][0:RMAX] for the tile's rows that have an adapter, 8 rows at a time per warp
// the adapter of row m (-1: none, or a scale of 0, or an adapter without this target)
__device__ __forceinline__ int row_adapter_id(const LoraArgs& p, const LoraOperands& ops, int64_t m) {
    if (m >= p.M) return -1;
    const int64_t e = m / p.rpe;
    const int id = p.row_adapter[e];
    if (id < 0 || id >= PB200_LORA_MAX_ADAPTERS || ops.op[id].rank_pad == 0 || p.row_scale[e] == 0.f) return -1;
    return id;
}

// the smallest adapter id among the tile's rows above prev (INT_MAX: none)
__device__ __forceinline__ int next_adapter(const int* id_s, int prev) {
    int cur = INT_MAX;
    for (int i = 0; i < LORA_TM; ++i) {
        const int v = id_s[i];
        if (v > prev && v < cur) cur = v;
    }
    return cur;
}

template <int RJ, bool LN>
__global__ void __launch_bounds__(LORA_THREADS) lora_shrink_kernel(const LoraArgs p, const __grid_constant__ LoraOperands ops) {
    constexpr int RMAX = LORA_WARPS * RJ;       // ranks this instance covers
    __shared__ int id_s[LORA_TM];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t row0 = (int64_t)blockIdx.x * LORA_TM;
    if (tid < LORA_TM) id_s[tid] = row_adapter_id(p, ops, row0 + tid);
    __syncthreads();
    for (int prev = -1;;) {
        const int cur = next_adapter(id_s, prev);
        if (cur == INT_MAX) break;
        prev = cur;
        const __half* const a = ops.op[cur].a;
        const float* const aux = ops.op[cur].aux;
        const int rp = ops.op[cur].rank_pad;
        for (int g = 0; g < LORA_TM / 8; ++g) {
            bool any = false;
#pragma unroll
            for (int r = 0; r < 8; ++r) any |= id_s[g * 8 + r] == cur;
            if (!any) continue;
            float acc[8][RJ];
#pragma unroll
            for (int r = 0; r < 8; ++r)
#pragma unroll
                for (int q = 0; q < RJ; ++q) acc[r][q] = 0.f;
            for (int k = lane * 8; k < p.K; k += 256) {
                float af[RJ][8];
#pragma unroll
                for (int q = 0; q < RJ; ++q) {
                    const int j = warp * RJ + q;
                    const uint4 v = j < rp ? __ldg(reinterpret_cast<const uint4*>(a + (int64_t)j * p.K + k)) : make_uint4(0, 0, 0, 0);
                    unpack8(v, af[q]);
                }
                uint4 xv[8];
#pragma unroll
                for (int r = 0; r < 8; ++r) {
                    xv[r] = make_uint4(0, 0, 0, 0);
                    if (id_s[g * 8 + r] == cur) xv[r] = __ldg(reinterpret_cast<const uint4*>(p.x + (row0 + g * 8 + r) * p.ldx + k));
                }
#pragma unroll
                for (int r = 0; r < 8; ++r) {
                    float xf[8];
                    unpack8(xv[r], xf);
#pragma unroll
                    for (int e = 0; e < 8; ++e)
#pragma unroll
                        for (int q = 0; q < RJ; ++q) acc[r][q] = fmaf(xf[e], af[q][e], acc[r][q]);
                }
            }
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                if (id_s[g * 8 + r] != cur) continue;
                const int64_t m = row0 + g * 8 + r;
                float neg_mean = 0.f, rstd = 1.f;
                if constexpr (LN) ln_stat_moments(p.ln_stat + 2 * m, p.K, neg_mean, rstd);   // as the PB200_EPI_F16_LN epilogue
#pragma unroll
                for (int q = 0; q < RJ; ++q) {
                    const float v = warp_sum(acc[r][q]);
                    const int j = warp * RJ + q;
                    if (lane == 0) {
                        float u = 0.f;
                        if (j < rp) u = LN ? fmaf(neg_mean, aux[j], v) * rstd : v;
                        p.u[m * RMAX + j] = u;
                    }
                }
            }
        }
    }
}

// ---- expand: y[o, n] += s * (alpha/r) * sum_j u[j] B[n, j] over a chunk of LORA_NCHUNK columns, two per thread
template <int RJ, bool F32>
__global__ void __launch_bounds__(LORA_THREADS) lora_expand_kernel(const LoraArgs p, const __grid_constant__ LoraOperands ops) {
    constexpr int RMAX = LORA_WARPS * RJ;
    __shared__ __align__(16) float u_s[LORA_TM][RMAX];
    __shared__ int id_s[LORA_TM];
    __shared__ float s_s[LORA_TM];
    const int tid = threadIdx.x;
    const int64_t row0 = (int64_t)blockIdx.x * LORA_TM;
    if (tid < LORA_TM) {
        id_s[tid] = row_adapter_id(p, ops, row0 + tid);
        s_s[tid] = id_s[tid] >= 0 ? p.row_scale[(row0 + tid) / p.rpe] : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < LORA_TM * RMAX; i += LORA_THREADS) {
        const int r = i / RMAX;
        if (id_s[r] >= 0) u_s[r][i % RMAX] = p.u[(row0 + r) * RMAX + i % RMAX];
    }
    __syncthreads();
    const int n = blockIdx.y * LORA_NCHUNK + 2 * tid;
    if (n >= p.N) return;
    for (int prev = -1;;) {
        const int cur = next_adapter(id_s, prev);
        if (cur == INT_MAX) break;
        prev = cur;
        const LoraOperand& op = ops.op[cur];
        const int rp = op.rank_pad;
        __half2 bh[RMAX];           // (B[n, j], B[n + 1, j])
#pragma unroll
        for (int q = 0; q < RMAX / 8; ++q) {
            uint4 v0 = make_uint4(0, 0, 0, 0), v1 = make_uint4(0, 0, 0, 0);
            if (q * 8 < rp) {
                v0 = __ldg(reinterpret_cast<const uint4*>(op.b + (int64_t)n * rp + q * 8));
                v1 = __ldg(reinterpret_cast<const uint4*>(op.b + (int64_t)(n + 1) * rp + q * 8));
            }
            const __half* h0 = reinterpret_cast<const __half*>(&v0);
            const __half* h1 = reinterpret_cast<const __half*>(&v1);
#pragma unroll
            for (int e = 0; e < 8; ++e) bh[q * 8 + e] = __halves2half2(h0[e], h1[e]);
        }
        const float alpha_r = op.aux[rp];
        for (int r0 = 0; r0 < LORA_TM; r0 += 8) {
            // the rows' y pairs are loaded together, so that eight loads are in flight per thread
            float2 yv[8];
            int64_t off[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int64_t m = row0 + r0 + i;
                off[i] = (p.remap_in > 0 ? (m / p.remap_in) * p.remap_out + m % p.remap_in : m) * p.ldy + n;
                if (id_s[r0 + i] != cur) continue;
                if constexpr (F32) yv[i] = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.y) + off[i]);
                else yv[i] = __half22float2(*reinterpret_cast<const __half2*>(reinterpret_cast<const __half*>(p.y) + off[i]));
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (id_s[r0 + i] != cur) continue;
                float a0 = 0.f, a1 = 0.f;
#pragma unroll
                for (int j = 0; j < RMAX; j += 4) {
                    const float4 u = *reinterpret_cast<const float4*>(&u_s[r0 + i][j]);
                    const float uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 b = __half22float2(bh[j + e]);
                        a0 = fmaf(uu[e], b.x, a0);
                        a1 = fmaf(uu[e], b.y, a1);
                    }
                }
                const float f = s_s[r0 + i] * alpha_r;
                if constexpr (F32) {
                    *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.y) + off[i]) = make_float2(yv[i].x + f * a0, yv[i].y + f * a1);
                } else {
                    *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.y) + off[i]) = __floats2half2_rn(yv[i].x + f * a0, yv[i].y + f * a1);
                }
            }
        }
    }
}

template <int RJ>
static int lora_dispatch(bool ln, bool f32, const LoraArgs& a, const LoraOperands& ops, cudaStream_t st) {
    const dim3 grid((unsigned)ceil_div(a.M, LORA_TM)), grid2(grid.x, (unsigned)ceil_div(a.N, LORA_NCHUNK));
    if (ln) lora_shrink_kernel<RJ, true><<<grid, LORA_THREADS, 0, st>>>(a, ops);
    else lora_shrink_kernel<RJ, false><<<grid, LORA_THREADS, 0, st>>>(a, ops);
    PB_LAUNCH_CHECK();
    if (f32) lora_expand_kernel<RJ, true><<<grid2, LORA_THREADS, 0, st>>>(a, ops);
    else lora_expand_kernel<RJ, false><<<grid2, LORA_THREADS, 0, st>>>(a, ops);
    PB_LAUNCH_CHECK();
    return 0;
}

int launch_lora(const __half* x, int64_t ldx, int64_t M, int K, int N, int rows_per_entry, const int* row_adapter,
                const float* row_scale, const LoraOperands& ops, const int64_t* ln_stat, void* y, int64_t ldy, bool y_f32,
                int remap_in, int remap_out, float* u_ws, cudaStream_t st) {
    if (M <= 0 || N <= 0) return 0;
    PB_CHECK(x && y && row_adapter && row_scale && u_ws, "lora: x, y, row_adapter, row_scale and the U scratch are required");
    PB_CHECK(N % 2 == 0 && ldy % 2 == 0 && ((uintptr_t)y & 7) == 0, "lora: N=%d and ldy=%lld must be even, y 8-byte aligned", N,
             (long long)ldy);
    PB_CHECK(K > 0 && K % 8 == 0 && ldx >= K && ldx % 8 == 0 && ((uintptr_t)x & 15) == 0,
             "lora: K=%d, ldx=%lld (multiples of 8, 16-byte aligned rows)", K, (long long)ldx);
    PB_CHECK(ldy >= N && rows_per_entry > 0 && remap_in >= 0 && (remap_in == 0 || remap_out >= remap_in),
             "lora: ldy=%lld for N=%d, rows_per_entry=%d, remap %d->%d", (long long)ldy, N, rows_per_entry, remap_in, remap_out);
    int max_rp = 0;
    for (int i = 0; i < PB200_LORA_MAX_ADAPTERS; ++i) {
        const LoraOperand& o = ops.op[i];
        if (o.rank_pad == 0) continue;
        PB_CHECK(o.rank_pad % 8 == 0 && o.rank_pad <= LORA_MAX_RANK && o.a && o.b && o.aux && ((uintptr_t)o.a & 15) == 0 &&
                     ((uintptr_t)o.b & 15) == 0, "lora: adapter %d: padded rank %d (8..64, multiple of 8), 16-byte aligned A and B",
                 i, o.rank_pad);
        max_rp = o.rank_pad > max_rp ? o.rank_pad : max_rp;
    }
    if (max_rp == 0) return 0;
    LoraArgs a{x, ldx, M, K, N, rows_per_entry, row_adapter, row_scale, ln_stat, u_ws, y, ldy, remap_in, remap_out};
    // an upper bound on the bytes: every row of the launch as if it had an adapter (x read once, y read and written once); which
    // rows have one is in a device table the host does not read
    ProfScope prof("lora", (double)M * ((double)K * 2.0 + (double)N * (y_f32 ? 8.0 : 4.0)), st);
    const int rj = max_rp / LORA_WARPS;
    if (rj <= 1) return lora_dispatch<1>(ln_stat != nullptr, y_f32, a, ops, st);
    if (rj <= 2) return lora_dispatch<2>(ln_stat != nullptr, y_f32, a, ops, st);
    if (rj <= 4) return lora_dispatch<4>(ln_stat != nullptr, y_f32, a, ops, st);
    return lora_dispatch<8>(ln_stat != nullptr, y_f32, a, ops, st);
}

}  // namespace pb

extern "C" int pb200_lora_shrink_expand(const void* x, int64_t ldx, int64_t m, int k, int n, int rows_per_entry, const int* row_adapter,
                                        const float* row_scale, const pb200_lora_operand* ops, int n_ops, const int64_t* ln_stat, void* y,
                                        int64_t ldy, int y_f32, int remap_in, int remap_out, void* workspace, int64_t workspace_bytes,
                                        void* stream) {
    PB_CHECK(workspace_bytes >= m * PB200_LORA_WORKSPACE_PER_ROW && ((uintptr_t)workspace & 15) == 0,
             "lora_shrink_expand: workspace of %lld bytes, %lld needed (16-byte aligned)", (long long)workspace_bytes,
             (long long)(m * PB200_LORA_WORKSPACE_PER_ROW));
    PB_CHECK(n_ops >= 0 && n_ops <= PB200_LORA_MAX_ADAPTERS && (n_ops == 0 || ops != nullptr), "lora_shrink_expand: %d adapters (0..%d)",
             n_ops, PB200_LORA_MAX_ADAPTERS);
    pb::LoraOperands o;
    memset(&o, 0, sizeof(o));
    for (int i = 0; i < n_ops; ++i)
        o.op[i] = pb::LoraOperand{reinterpret_cast<const __half*>(ops[i].a), reinterpret_cast<const __half*>(ops[i].b), ops[i].aux,
                                  ops[i].rank_pad};
    return pb::launch_lora(reinterpret_cast<const __half*>(x), ldx, m, k, n, rows_per_entry, row_adapter, row_scale, o, ln_stat, y, ldy,
                           y_f32 != 0, remap_in, remap_out, reinterpret_cast<float*>(workspace), (cudaStream_t)stream);
}
