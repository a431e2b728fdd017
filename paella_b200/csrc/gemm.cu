// wgmma GEMM for every Linear / 1x1-conv / patchify contraction on the path:
//     C[M,N] = A[M,K] . W[N,K]^T   (fp16 operands, fp32 accumulation in registers)  + fused epilogue
// Replaces the cuBLAS/cuDNN calls behind nn.Linear / nn.Conv2d(k=1) / Conv2d(k=2,s=2) /
// ConvTranspose2d(k=2,s=2) in ref/src/modules.py (ResBlock :49-55, AttnBlock :71-74, embedding :130-134,
// resamplers :153-156,172-175, clf/out_mapper :179-187) and ref/src/vqgan.py (ResBlock :16-20).
//
// One persistent, warp-specialised kernel (gemm_f16_kernel), M128 x N{64,128,256} tiles, 384 threads:
//   warpgroup 0    : TMA producer  - one thread issues cp.async.bulk.tensor loads of the 128x64 A tile and the BLOCK_N x 64
//                    W tile, 128B-swizzled, into a 3-8 stage shared-memory ring guarded by full/empty mbarriers; the
//                    warpgroup hands its registers to the MMA warpgroups (setmaxnreg)
//   warpgroups 1,2 : MMA + epilogue - each issues wgmma m64nNk16 (4 per stage) for its 64 rows of the tile, keeps one
//                    k-block in flight and releases the previous stage; then the fused epilogue (bias / GELU + GRN statistic /
//                    residual + FiLM / LayerNorm fold / un-patchify / NCHW transpose) through a shared-memory slab that turns
//                    the accumulator fragment into row-per-lane chunks, transposed inside the warp so that every store
//                    instruction writes whole 128-byte lines.  The producer runs ahead into the next tile meanwhile.
// Scheduling: tile width from a tensor / L2 cycle model (gemm_pick_block_n), programmatic dependent launch so the prologue
// overlaps the previous kernel.
#include "gemm.cuh"
#include <type_traits>

#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <unordered_map>

namespace pb {

// ------------------------------------------------------------------ tensor maps (host)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    });
    return fn;
}

int make_tmap_f16_2d(CUtensorMap* tm, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
    EncodeTiledFn fn = encode_fn();
    PB_CHECK(fn != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
    PB_CHECK(((uintptr_t)ptr & 15) == 0, "TMA: base pointer must be 16-byte aligned");
    PB_CHECK((ld * 2) % 16 == 0, "TMA: row stride %lld halves is not a multiple of 16 bytes", (long long)ld);
    PB_CHECK(box_rows >= 1 && box_rows <= 256, "TMA: bad box rows %d", box_rows);
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)(ld * 2)};
    cuuint32_t box[2] = {(cuuint32_t)GEMM_BLOCK_K, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld box_rows=%d", (int)r,
             (long long)rows, (long long)cols, (long long)ld, box_rows);
    return 0;
}

// 2-D fp16 tensor map with an explicit box and swizzle: swizzle_bytes = 128 (box_cols <= 64) or 32 (box_cols <= 16)
int make_tmap_f16_2d_box(CUtensorMap* tm, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows,
                         int swizzle_bytes) {
    EncodeTiledFn fn = encode_fn();
    PB_CHECK(fn != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
    PB_CHECK(((uintptr_t)ptr & 15) == 0, "TMA: base pointer must be 16-byte aligned");
    PB_CHECK((ld * 2) % 16 == 0, "TMA: row stride %lld halves is not a multiple of 16 bytes", (long long)ld);
    PB_CHECK(swizzle_bytes == 128 || swizzle_bytes == 64 || swizzle_bytes == 32 || swizzle_bytes == 0, "TMA: swizzle %d unsupported", swizzle_bytes);
    PB_CHECK(box_rows >= 1 && box_rows <= 256 && box_cols >= 8 && (swizzle_bytes == 0 ? box_cols <= 256 : box_cols * 2 <= swizzle_bytes),
             "TMA: bad box %dx%d for swizzle %d", box_rows, box_cols, swizzle_bytes);
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)(ld * 2)};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                    : (swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE),
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(box %dx%d, swizzle %d) failed (%d)", box_rows, box_cols, swizzle_bytes, (int)r);
    return 0;
}

// Tensor maps are pure functions of (pointer, shape, box): the executors' workspaces are bump-allocated identically every call
// and the weights never move, so a process-wide cache removes the driver call from all but the first launches.
int cached_tmap_f16_2d(const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows, int swizzle_bytes,
                       CUtensorMap* out) {
    using Key = std::tuple<const void*, int64_t, int64_t, int64_t, int, int, int>;
    static std::map<Key, CUtensorMap> cache;
    static std::mutex mu;
    const Key key{ptr, rows, cols, ld, box_cols, box_rows, swizzle_bytes};
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(key);
    if (it == cache.end()) {
        if (cache.size() > 8192) cache.clear();
        CUtensorMap tm;
        PB_TRY(make_tmap_f16_2d_box(&tm, ptr, rows, cols, ld, box_cols, box_rows, swizzle_bytes));
        it = cache.emplace(key, tm).first;
    }
    *out = it->second;
    return 0;
}

// rank-N fp16 tensor map (dims/strides innermost first, strides in bytes for dims 1..rank-1), 128-byte swizzle
int make_tmap_f16_nd(CUtensorMap* tm, const void* ptr, int rank, const int64_t* dims, const int64_t* strides_bytes,
                     const int* box) {
    EncodeTiledFn fn = encode_fn();
    PB_CHECK(fn != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
    PB_CHECK(rank >= 2 && rank <= 5, "TMA: rank %d unsupported", rank);
    PB_CHECK(((uintptr_t)ptr & 15) == 0, "TMA: base pointer must be 16-byte aligned");
    cuuint64_t d[5], s[4];
    cuuint32_t b[5], e[5];
    for (int i = 0; i < rank; ++i) {
        d[i] = (cuuint64_t)dims[i];
        b[i] = (cuuint32_t)box[i];
        e[i] = 1;
        PB_CHECK(box[i] >= 1 && box[i] <= 256, "TMA: bad box[%d]=%d", i, box[i]);
        if (i > 0) {
            PB_CHECK(strides_bytes[i - 1] % 16 == 0, "TMA: stride %lld not a multiple of 16 bytes", (long long)strides_bytes[i - 1]);
            s[i - 1] = (cuuint64_t)strides_bytes[i - 1];
        }
    }
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), d, s, b, e,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(rank %d) failed (%d)", rank, (int)r);
    return 0;
}

// ------------------------------------------------------------------ epilogue
// Global operands of a 32-column chunk that do not depend on the accumulator (the fp32 residual row segment).  They
// are fetched for the whole chunk BEFORE its store loop: out may alias resid (the model updates x in place), so inside
// the store loop the compiler must order every load after the previous store -- 8 dependent L2 round trips per chunk
// instead of 8 independent loads in flight together.
template <int MODE>
struct EpiPre {};
template <>
struct EpiPre<PB200_EPI_RESID_F32> { float4 r[8]; };
template <>
struct EpiPre<PB200_EPI_F16_LN> { float neg_mean = 0.f, rstd = 0.f; };     // this lane's row, computed once per tile
template <>
struct EpiPre<PB200_EPI_RESID_LN_F32> {
    float4 r[8];
    float ln_s = 0.f, ln_q = 0.f;      // this lane's row: sum / sum of squares over the chunks of the tile done so far
    float shift = 0.f;                 // this lane's row: the shift subtracted before the fp16 copy and the statistics
};

// Coalescing.  The epilogue hands every lane one ROW of the chunk (32 consecutive columns), so a direct 16-byte store
// per lane touches 32 different 128-byte lines per instruction and the LSU serialises them.  The chunk is therefore transposed inside the
// warp with xor-butterfly shuffles first:
//   fp32: 8x8 transpose of float4 items in 8-lane groups -> lane (a,b) item i = row 8a+i, columns 4b..4b+3
//         (a store instruction then writes 4 full 128-byte lines);
//   fp16: 4x4 transpose of 8-half items in 4-lane groups -> lane (a,b) item i = row 4a+i, columns 8b..8b+7
//         (8 rows x 64 contiguous bytes per instruction).
__device__ __forceinline__ void transpose4x4_u4(uint32_t (&pk)[16], int lane) {
#pragma unroll
    for (int s = 2; s > 0; s >>= 1) {
        const bool up = (lane & s) != 0;
#pragma unroll
        for (int g0 = 0; g0 < 4; ++g0) {
            if (g0 & s) continue;
            const int g1 = g0 | s;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const uint32_t send = up ? pk[g0 * 4 + e] : pk[g1 * 4 + e];
                const uint32_t recv = __shfl_xor_sync(0xffffffffu, send, s);
                if (up) pk[g0 * 4 + e] = recv;
                else pk[g1 * 4 + e] = recv;
            }
        }
    }
}
// fp16 row-per-lane chunk -> transposed, coalesced store.  `orow` is this lane's output row (or -1 if masked).
__device__ __forceinline__ void store_chunk_f16(const float (&v)[32], __half* out, int64_t ldo, int64_t orow, int col0,
                                                int N, int lane) {
    uint32_t pk[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) pk[j] = pack_half2(v[2 * j], v[2 * j + 1]);
    transpose4x4_u4(pk, lane);
    const int col = col0 + (lane & 3) * 8;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t r = __shfl_sync(0xffffffffu, orow, (lane & 28) + i);
        if (r >= 0 && col < N)
            *reinterpret_cast<uint4*>(out + r * ldo + col) = make_uint4(pk[i * 4], pk[i * 4 + 1], pk[i * 4 + 2], pk[i * 4 + 3]);
    }
}

template <int MODE>
__device__ __forceinline__ void epilogue_preload(const pb200_gemm_epilogue& ep, int M, int N, int row, int col0,
                                                 EpiPre<MODE>& pre, int lane, bool first_chunk) {
    if constexpr (MODE == PB200_EPI_F16_LN) {
        if (first_chunk && row < M) {      // row statistics -> (mean, rstd), once per tile
            const longlong2 st = *reinterpret_cast<const longlong2*>(ep.ln_stat + 2 * (int64_t)row);
            const float inv_c = 1.0f / (float)ep.ln_c;
            const float mean = (float)st.x * (1.0f / 1048576.0f) * inv_c;
            const float ex2 = (float)st.y * (1.0f / 65536.0f) * inv_c;
            pre.neg_mean = -mean;
            pre.rstd = 1.0f / sqrtf(fmaxf(ex2 - mean * mean, 0.f) + 1e-6f);
            // the true row mean, for the next producer's shift (every N-tile writes the same value: benign)
            if (ep.ln_mean_out) ep.ln_mean_out[row] = (ep.ln_shift ? ep.ln_shift[row] : 0.f) + mean;
        }
    }
    if constexpr (MODE == PB200_EPI_RESID_LN_F32) {
        if (first_chunk) pre.shift = (ep.ln_shift && row < M) ? ep.ln_shift[row] : 0.f;
    }
    if constexpr (MODE == PB200_EPI_RESID_F32 || MODE == PB200_EPI_RESID_LN_F32) {
        const int col = col0 + (lane & 7) * 4;       // transposed layout: item i = row of lane (lane & 24) + i
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = __shfl_sync(0xffffffffu, row, (lane & 24) + i);
            if (r < M && col < N) pre.r[i] = *reinterpret_cast<const float4*>(ep.resid + (int64_t)r * ep.ldr + col);
        }
    }
}

template <int MODE>
__device__ __forceinline__ void epilogue_chunk(const pb200_gemm_epilogue& ep, int M, int N, int row, int col0,
                                               float (&v)[32], int lane, EpiPre<MODE>& pre) {
    const bool row_ok = row < M;
    // warp-uniform: no column / row of this chunk is out of range -> the hot path carries no per-element predicates
    const bool full_cols = col0 + 32 <= N;
    const bool full = full_cols && __all_sync(0xffffffffu, row_ok);
    // ---- folded LayerNorm of the A rows: acc = x W^T with x un-normalised; LN(x) W^T = rstd (acc - mean rowsum(W))
    if constexpr (MODE == PB200_EPI_F16_LN) {
        const float nm = pre.neg_mean, rstd = pre.rstd;
#pragma unroll
        for (int g = 0; g < 8; ++g) {
            if (col0 + g * 4 < N) {
                const float4 ws = __ldg(reinterpret_cast<const float4*>(ep.ln_wsum + col0 + g * 4));
                v[g * 4 + 0] = fmaf(nm, ws.x, v[g * 4 + 0]) * rstd; v[g * 4 + 1] = fmaf(nm, ws.y, v[g * 4 + 1]) * rstd;
                v[g * 4 + 2] = fmaf(nm, ws.z, v[g * 4 + 2]) * rstd; v[g * 4 + 3] = fmaf(nm, ws.w, v[g * 4 + 3]) * rstd;
            }
        }
    }
    // ---- bias (indexed by GEMM column in every mode)
    if (ep.bias) {
        if (full_cols) {
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                const float4 b = __ldg(reinterpret_cast<const float4*>(ep.bias + col0 + g * 4));
                v[g * 4 + 0] += b.x; v[g * 4 + 1] += b.y; v[g * 4 + 2] += b.z; v[g * 4 + 3] += b.w;
            }
        } else {
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                if (col0 + g * 4 < N) {
                    const float4 b = __ldg(reinterpret_cast<const float4*>(ep.bias + col0 + g * 4));
                    v[g * 4 + 0] += b.x; v[g * 4 + 1] += b.y; v[g * 4 + 2] += b.z; v[g * 4 + 3] += b.w;
                }
            }
        }
    }
    if (MODE == PB200_EPI_F16 || MODE == PB200_EPI_F32 || MODE == PB200_EPI_F16_LN) {
        int64_t orow = row_ok ? row : -1;
        if (row_ok && ep.remap_in > 0) orow = (int64_t)(row / ep.remap_in) * ep.remap_out + (row % ep.remap_in);
        if (MODE == PB200_EPI_F16 || MODE == PB200_EPI_F16_LN) {
            store_chunk_f16(v, reinterpret_cast<__half*>(ep.out), ep.ldo, orow, col0, N, lane);
        } else {
            transpose8x8_f4(v, lane);
            const int col = col0 + (lane & 7) * 4;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int64_t r = __shfl_sync(0xffffffffu, orow, (lane & 24) + i);
                if (r >= 0 && col < N)
                    *reinterpret_cast<float4*>(reinterpret_cast<float*>(ep.out) + r * ep.ldo + col) =
                        make_float4(v[i * 4], v[i * 4 + 1], v[i * 4 + 2], v[i * 4 + 3]);
            }
        }
    } else if (MODE == PB200_EPI_GELU_F16) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = gelu_erf_fast(v[j]);
        store_chunk_f16(v, reinterpret_cast<__half*>(ep.out), ep.ldo, row_ok ? (int64_t)row : -1, col0, N, lane);
        if (ep.sqsum) {   // GlobalResponseNorm statistic: sum over the sample's positions of h^2, per channel.
            // Accumulated in 2^-24 fixed point with 64-bit integer atomics: integer addition is associative, so the
            // result does not depend on the order in which warps/CTAs arrive (float atomics made two runs of the same
            // seed differ in the last bits, which flipped ~2% of the sampled tokens over 8 steps).
            unsigned long long* sq = reinterpret_cast<unsigned long long*>(ep.sqsum);
            auto fx = [](float x) { return (unsigned long long)__float2ull_rn(x * 16777216.0f); };
            const int P = ep.rows_per_sample;
            if (full) {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] *= v[j];
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] = (row_ok && col0 + j < N) ? v[j] * v[j] : 0.f;
            }
            if ((P & 31) == 0) {
                // transpose-reduce over the warp's 32 rows: lane j ends with the column-(col0+j) sum
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
                    for (int i = 0; i < o; ++i) {
                        const bool up = (lane & o) != 0;
                        const float send = up ? v[i] : v[i + o];
                        const float keep = up ? v[i + o] : v[i];
                        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
                    }
                }
                const int row0 = row - lane;
                if (row0 < M && col0 + lane < N)
                    atomicAdd(sq + (int64_t)(row0 / P) * N + col0 + lane, fx(v[0]));
            } else if (P == 16 || P == 8 || P == 4 || P == 2) {
                // the warp's 32 rows hold 32/P whole samples: the same transpose-reduce inside aligned groups of P
                // lanes, on 32/P sets of P columns -> lane l ends with columns {j*P + (l % P)} of its group's sample
                // (~30 shuffles and 32/P atomics per lane instead of 32 x log2(P) shuffles and 32 atomics)
                auto grouped = [&](auto pc) {
                    constexpr int PP = decltype(pc)::value;
#pragma unroll
                    for (int o = PP / 2; o > 0; o >>= 1) {
                        const bool up = (lane & o) != 0;
#pragma unroll
                        for (int j = 0; j < 32 / PP; ++j)
#pragma unroll
                            for (int i = 0; i < o; ++i) {
                                const float send = up ? v[j * PP + i] : v[j * PP + i + o];
                                const float keep = up ? v[j * PP + i + o] : v[j * PP + i];
                                v[j * PP + i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
                            }
                    }
                    const int grow = row - (lane & (PP - 1));          // first row of this lane's sample
                    if (grow < M) {
#pragma unroll
                        for (int j = 0; j < 32 / PP; ++j) {
                            const int col = col0 + j * PP + (lane & (PP - 1));
                            if (col < N) atomicAdd(sq + (int64_t)(grow / PP) * N + col, fx(v[j * PP]));
                        }
                    }
                };
                if (P == 16) grouped(std::integral_constant<int, 16>{});
                else if (P == 8) grouped(std::integral_constant<int, 8>{});
                else if (P == 4) grouped(std::integral_constant<int, 4>{});
                else grouped(std::integral_constant<int, 2>{});
            } else if (row_ok) {
#pragma unroll
                for (int j = 0; j < 32; ++j)
                    if (col0 + j < N) atomicAdd(sq + (int64_t)(row / P) * N + col0 + j, fx(v[j]));
            }
        }
    } else if (MODE == PB200_EPI_RESID_F32 || MODE == PB200_EPI_RESID_LN_F32) {
        // (bias was added above in the row-per-lane layout); the rest runs in the transposed, coalesced layout
        transpose8x8_f4(v, lane);
        const int col = col0 + (lane & 7) * 4;
        float* obase = reinterpret_cast<float*>(ep.out);
        float ls[8], lq[8], sh[8];
        if constexpr (MODE == PB200_EPI_RESID_LN_F32) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                ls[i] = lq[i] = 0.f;
                sh[i] = __shfl_sync(0xffffffffu, pre.shift, (lane & 24) + i);     // item i = the row of lane (lane & 24) + i
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = __shfl_sync(0xffffffffu, row, (lane & 24) + i);
            if (r < M && col < N) {
                float4 rr = make_float4(0.f, 0.f, 0.f, 0.f);
                if constexpr (MODE == PB200_EPI_RESID_F32 || MODE == PB200_EPI_RESID_LN_F32) rr = pre.r[i];
                float4 y;
                y.x = fmaf(v[i * 4 + 0], ep.alpha, rr.x); y.y = fmaf(v[i * 4 + 1], ep.alpha, rr.y);
                y.z = fmaf(v[i * 4 + 2], ep.alpha, rr.z); y.w = fmaf(v[i * 4 + 3], ep.alpha, rr.w);
                if (ep.film) {
                    const float* fa = ep.film + (int64_t)(r / ep.rows_per_sample) * ep.film_ld + ep.film_off + col;
                    const float4 a = __ldg(reinterpret_cast<const float4*>(fa));
                    const float4 b = __ldg(reinterpret_cast<const float4*>(fa + N));
                    y.x = fmaf(y.x, 1.0f + a.x, b.x); y.y = fmaf(y.y, 1.0f + a.y, b.y);
                    y.z = fmaf(y.z, 1.0f + a.z, b.z); y.w = fmaf(y.w, 1.0f + a.w, b.w);
                }
                *reinterpret_cast<float4*>(obase + (int64_t)r * ep.ldo + col) = y;
                if constexpr (MODE == PB200_EPI_RESID_LN_F32) {
                    y.x -= sh[i]; y.y -= sh[i]; y.z -= sh[i]; y.w -= sh[i];      // (after the fp32 store of the true value)
                    uint2 pk;
                    pk.x = pack_half2(y.x, y.y);
                    pk.y = pack_half2(y.z, y.w);
                    *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(ep.out16) + (int64_t)r * ep.ldo + col) = pk;
                    ls[i] = (y.x + y.y) + (y.z + y.w);
                    lq[i] = (y.x * y.x + y.y * y.y) + (y.z * y.z + y.w * y.w);
                }
            }
        }
        if constexpr (MODE == PB200_EPI_RESID_LN_F32) {
            // row statistics of the finished rows: item i of lane (a,b) is row 8a+i, columns 4b..4b+3 -> transpose-reduce
            // over the 8 lanes of the group; lane 8a+b ends with the sums of row 8a+b, i.e. of its own `row`
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) {
                const bool up = (lane & o) != 0;
#pragma unroll
                for (int i = 0; i < o; ++i) {
                    const float s_send = up ? ls[i] : ls[i + o], s_keep = up ? ls[i + o] : ls[i];
                    const float q_send = up ? lq[i] : lq[i + o], q_keep = up ? lq[i + o] : lq[i];
                    ls[i] = s_keep + __shfl_xor_sync(0xffffffffu, s_send, o);
                    lq[i] = q_keep + __shfl_xor_sync(0xffffffffu, q_send, o);
                }
            }
            pre.ln_s += ls[0];          // flushed once per tile by epilogue_finish (one atomic pair per row and warp)
            pre.ln_q += lq[0];
        }
    } else if (MODE == PB200_EPI_UNPATCH_F32) {
        if (!row_ok) return;
        const int hw = ep.up_h * ep.up_w;
        const int b = row / hw, rem = row - b * hw;
        const int y = rem / ep.up_w, x = rem - y * ep.up_w;
        float* obase = reinterpret_cast<float*>(ep.out);
#pragma unroll
        for (int g = 0; g < 8; ++g) {
            const int col = col0 + g * 4;
            if (col < N) {
                const int q = col / ep.up_cout, co = col - q * ep.up_cout;    // q = dy*2+dx
                const int64_t orow = ((int64_t)b * 2 * ep.up_h + 2 * y + (q >> 1)) * (2 * ep.up_w) + 2 * x + (q & 1);
                *reinterpret_cast<float4*>(obase + orow * ep.up_cout + co) =
                    make_float4(v[g * 4], v[g * 4 + 1], v[g * 4 + 2], v[g * 4 + 3]);
            }
        }
    } else if (MODE == PB200_EPI_NCHW_F32) {
        if (!row_ok) return;
        const int hw = ep.rows_per_sample;
        const int b = row / hw, p = row - b * hw;
        float* o = reinterpret_cast<float*>(ep.out) + ((int64_t)b * N + col0) * hw + p;
#pragma unroll
        for (int j = 0; j < 32; ++j)
            if (col0 + j < N) o[(int64_t)j * hw] = v[j];
    }
}

// after the last chunk of a tile: flush what the chunks accumulated per row
template <int MODE>
__device__ __forceinline__ void epilogue_finish(const pb200_gemm_epilogue& ep, int M, int row, EpiPre<MODE>& pre) {
    if constexpr (MODE == PB200_EPI_RESID_LN_F32) {
        if (row < M) {
            unsigned long long* st = reinterpret_cast<unsigned long long*>(ep.ln_stat) + 2 * (int64_t)row;
            atomicAdd(st, (unsigned long long)__float2ll_rn(pre.ln_s * 1048576.0f));
            atomicAdd(st + 1, (unsigned long long)__float2ll_rn(pre.ln_q * 65536.0f));
        }
    }
}

// ------------------------------------------------------------------ kernel
// AMODE 0: A is a [M,K] matrix.  AMODE 1/2: A rows are gathered by TMA straight from an NHWC fp16 activation
// (im2col-free convolution): a 128-row tile is a th x tw patch of the output grid and k-block kb selects a filter
// tap and a 64-channel slice; out-of-image taps are zero-filled by the TMA unit (the conv's zero padding).
// ASCALE (GlobalResponseNorm folded into the A operand, ref/src/modules.py:37-40 + :53): the A tile is multiplied in shared
// memory, between TMA and MMA, by a per-(sample, k) fp16 factor  s[b, k] = 1 + gamma[k] * Nx[b, k]  -- GEMM2 of a ResBlock then
// computes (h * s) W2^T + (W2 beta + b2) = GRN(h) W2^T + b2 without the separate read-modify-write pass over the 4c-wide hidden.
// The [samples x 64] slice of s lands in the stage beside A and W; each MMA warpgroup rescales its own 64 rows in place (one
// HMUL2 rounding, the fp16 product), fences the generic->async proxy and only then issues its wgmma.
template <int BLOCK_N, int MODE, int AMODE, bool ASCALE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                const __grid_constant__ CUtensorMap tm_s, const pb200_gemm_epilogue ep, const ConvGeom geom, int M, int N,
                int K) {
    using L = GemmSmem<BLOCK_N, ASCALE>;
    constexpr int NSUB = BLOCK_N > 128 ? 2 : 1;          // a 256-wide tile is issued as two n128 wgmma per k-step
    constexpr int SUBN = BLOCK_N / NSUB;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    const uint32_t bar_base = smem_base + L::STAGES * L::STAGE_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (L::STAGES + s); };
    float* epi_stage = reinterpret_cast<float*>(smem_gen + L::STAGES * L::STAGE_BYTES + 256);

    const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
    const int lane = threadIdx.x & 31;
    const int n_tiles_n = (N + BLOCK_N - 1) / BLOCK_N;
    const int n_tiles_m = AMODE == 0 ? (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M : geom.batch * geom.tiles_y * geom.tiles_x;
    const int n_kb = (K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
    const int n_units = n_tiles_m * n_tiles_n;
    const int P = ep.rows_per_sample;
    const int ns = ASCALE ? (P >= GEMM_BLOCK_M ? 1 : GEMM_BLOCK_M / P) : 0;      // samples in a 128-row tile

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&tm_a);
        ptx::prefetch_tensormap(&tm_b);
        for (int s = 0; s < L::STAGES; ++s) {
            ptx::mbar_init(full_bar(s), 1);
            ptx::mbar_init(empty_bar(s), GEMM_CONSUMERS);      // one arrival per MMA warpgroup
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    // everything above overlapped the tail of the previous kernel (programmatic dependent launch); its results are
    // read from here on
    ptx::griddep_launch();
    ptx::griddep_wait();

    if (wg == 0) {
        // ===================== TMA producer (one elected thread of warp 0) =====================
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x < 32 && ptx::elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
                const int mt = unit / n_tiles_n;
                const int m_idx = mt * GEMM_BLOCK_M;
                const int n_idx = (unit % n_tiles_n) * BLOCK_N;
                int cb = 0, cy0 = 0, cx0 = 0;
                if (AMODE != 0) {
                    cb = mt / (geom.tiles_y * geom.tiles_x);
                    const int r = mt - cb * geom.tiles_y * geom.tiles_x;
                    cy0 = (r / geom.tiles_x) * geom.th;
                    cx0 = (r % geom.tiles_x) * geom.tw;
                }
                for (int kb = 0; kb < n_kb; ++kb) {
                    ptx::mbar_wait(empty_bar(stage), phase ^ 1);
                    ptx::mbar_arrive_expect_tx(full_bar(stage), (uint32_t)(L::A_BYTES + L::B_BYTES + ns * GEMM_BLOCK_K * 2));
                    const uint32_t sa = smem_base + stage * L::STAGE_BYTES;
                    if (AMODE == 0) {
                        ptx::tma_load_2d(&tm_a, full_bar(stage), sa, kb * GEMM_BLOCK_K, m_idx);
                    } else if (AMODE == 1) {
                        // Conv2d(k=4, s=2, p=1): tap (ky,kx) reads input (2y-1+ky, 2x-1+kx) = parity plane (pa,pb) at
                        // (y+a, x+b) of the [B, H/2, 2, W/2, 2*C] view
                        const int tap = kb / geom.n_cchunk, cc = kb - tap * geom.n_cchunk;
                        const int dy = (tap >> 2) - 1, dx = (tap & 3) - 1;
                        const int a = dy < 0 ? -1 : (dy >> 1), b = dx < 0 ? -1 : (dx >> 1);
                        const int pa = dy - 2 * a, pb = dx - 2 * b;
                        ptx::tma_load_5d(&tm_a, full_bar(stage), sa, pb * geom.cin + cc * 64, cx0 + b, pa, cy0 + a, cb);
                    } else {
                        // ConvTranspose2d(k=4, s=2, p=1), output phase (py,px): 2x2 taps at (y+oy, x+ox)
                        const int tap = kb / geom.n_cchunk, cc = kb - tap * geom.n_cchunk;
                        const int ty = tap >> 1, tx = tap & 1;
                        const int oy = geom.py == 0 ? (ty == 0 ? 0 : -1) : (ty == 0 ? 1 : 0);
                        const int ox = geom.px == 0 ? (tx == 0 ? 0 : -1) : (tx == 0 ? 1 : 0);
                        ptx::tma_load_4d(&tm_a, full_bar(stage), sa, cc * 64, cx0 + ox, cy0 + oy, cb);
                    }
                    // the W map's box is half a tile (BLOCK_N/2 rows): two loads
                    ptx::tma_load_2d(&tm_b, full_bar(stage), sa + L::A_BYTES, kb * GEMM_BLOCK_K, n_idx);
                    ptx::tma_load_2d(&tm_b, full_bar(stage), sa + L::A_BYTES + L::B_BYTES / 2, kb * GEMM_BLOCK_K,
                                     n_idx + BLOCK_N / 2);
                    if (ASCALE)
                        ptx::tma_load_2d(&tm_s, full_bar(stage), sa + L::A_BYTES + L::B_BYTES, kb * GEMM_BLOCK_K, m_idx / P);
                    if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== MMA + epilogue: warpgroup cw owns rows [64 cw, 64 cw + 64) of every tile =====================
        ptx::setmaxnreg_inc<232>();
        const int cw = wg - 1;
        const int tid = threadIdx.x & 127;
        const int wq = tid >> 5;                 // warp of the warpgroup: wgmma rows [16 wq, 16 wq + 16)
        float* stage_rows = epi_stage + cw * 64 * GEMM_EPI_STRIDE;
        float acc[NSUB][SUBN / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
            const int mt = unit / n_tiles_n;
            const int m_idx = mt * GEMM_BLOCK_M;
            const int n_idx = (unit % n_tiles_n) * BLOCK_N;
            int prev = 0;
            for (int kb = 0; kb < n_kb; ++kb) {
                ptx::mbar_wait(full_bar(stage), phase);
                const uint32_t sa = smem_base + stage * L::STAGE_BYTES;
                if (ASCALE) {
                    // thread = half a row: chunks [4 (tid & 1), +4) of row 64 cw + tid / 2; logical 16-byte chunk j of row r
                    // sits at j ^ (r & 7) (128-byte swizzle)
                    const int r = cw * 64 + (tid >> 1);
                    const int sl = P >= GEMM_BLOCK_M ? 0 : min(r / P, ns - 1);
                    uint8_t* sg = smem_gen + stage * L::STAGE_BYTES;
                    uint4* arow = reinterpret_cast<uint4*>(sg + r * 128);
                    const uint4* srow = reinterpret_cast<const uint4*>(sg + L::A_BYTES + L::B_BYTES + sl * 128);
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int j = (tid & 1) * 4 + jj;
                        uint4 av = arow[j ^ (r & 7)];
                        const uint4 sv = srow[j];
                        __half2* a2 = reinterpret_cast<__half2*>(&av);
                        const __half2* s2 = reinterpret_cast<const __half2*>(&sv);
#pragma unroll
                        for (int e = 0; e < 4; ++e) a2[e] = __hmul2(a2[e], s2[e]);
                        arow[j ^ (r & 7)] = av;
                    }
                    ptx::fence_proxy_async_smem();       // the rescaled rows must be visible to the tensor core's async proxy
                    ptx::bar_sync(1 + cw, 128);
                }
                const uint64_t da = ptx::wgmma_desc_kmajor_sw128(sa + (uint32_t)cw * (64 * 128));
                const uint64_t db = ptx::wgmma_desc_kmajor_sw128(sa + L::A_BYTES);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < GEMM_BLOCK_K / 16; ++k) {
                    // advance 16 elements (32 bytes) along K inside the 128-byte swizzle atom: +2 in (addr>>4)
                    const uint32_t accum = (kb | k) != 0 ? 1u : 0u;
#pragma unroll
                    for (int s = 0; s < NSUB; ++s) {
                        const uint64_t dbs = db + (uint64_t)((s * SUBN * 128) >> 4) + 2 * k;
                        if constexpr (SUBN == 64) ptx::wgmma_m64n64k16(acc[s], da + 2 * k, dbs, accum);
                        else ptx::wgmma_m64n128k16(acc[s], da + 2 * k, dbs, accum);
                    }
                }
                ptx::wgmma_commit();
                if (kb > 0) {              // the previous k-block's MMAs have retired: its stage goes back to the producer
                    ptx::wgmma_wait<1>();
                    if (tid == 0) ptx::mbar_arrive(empty_bar(prev));
                }
                prev = stage;
                if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
            }
            ptx::wgmma_wait<0>();
            if (tid == 0) ptx::mbar_arrive(empty_bar(prev));
#pragma unroll
            for (int s = 0; s < NSUB; ++s) ptx::fence_regs(acc[s]);

            // ---- epilogue.  The accumulator fragment (thread = rows 16 wq + lane/4 (+8), column pairs) goes through shared
            // memory in 64-column slabs so that the epilogue sees what it is written for: lane = row, 32 consecutive columns.
            // Warp wq takes rows [32 (wq & 1), +32) of the warpgroup's 64 and columns [32 (wq >> 1), +32) of the slab.
            const int rl = (wq & 1) * 32 + lane;               // row of the warpgroup's 64
            const int r = cw * 64 + rl;                         // row of the 128-row tile
            int row = m_idx + r;
            if (AMODE != 0) {   // tile row r = (ly, lx) of a th x tw patch -> output pixel row of the NHWC result
                const int cb = mt / (geom.tiles_y * geom.tiles_x);
                const int rr = mt - cb * geom.tiles_y * geom.tiles_x;
                const int gy = (rr / geom.tiles_x) * geom.th + r / geom.tw;
                const int gx = (rr % geom.tiles_x) * geom.tw + r % geom.tw;
                row = (gy < geom.gh && gx < geom.gw)
                          ? ((cb * geom.oh + gy * geom.sy + geom.py) * geom.ow + gx * geom.sx + geom.px)
                          : M;      // M = B*oh*ow: out of range -> masked
            }
            EpiPre<MODE> pre;
#pragma unroll 1
            for (int c64 = 0; c64 < BLOCK_N / 64; ++c64) {
                if (n_idx + c64 * 64 >= N) break;
                // the 32 registers of slab c64 (compile-time indices: one case per slab), each written once
                auto scatter = [&](auto slab) {
                    constexpr int C = decltype(slab)::value;
                    constexpr int S = (C * 64) / SUBN, I0 = ((C * 64) % SUBN) / 2;
#pragma unroll
                    for (int i = 0; i < 32; ++i)
                        stage_rows[(wq * 16 + (lane >> 2) + 8 * ((i >> 1) & 1)) * GEMM_EPI_STRIDE + (i >> 2) * 8 + 2 * (lane & 3) + (i & 1)] =
                            acc[S][I0 + i];
                };
                switch (c64) {
                    case 0: scatter(std::integral_constant<int, 0>{}); break;
                    case 1: if constexpr (BLOCK_N > 64) scatter(std::integral_constant<int, (BLOCK_N > 64 ? 1 : 0)>{}); break;
                    case 2: if constexpr (BLOCK_N > 128) scatter(std::integral_constant<int, (BLOCK_N > 128 ? 2 : 0)>{}); break;
                    default: if constexpr (BLOCK_N > 128) scatter(std::integral_constant<int, (BLOCK_N > 128 ? 3 : 0)>{}); break;
                }
                ptx::bar_sync(1 + cw, 128);
                const int col0 = n_idx + c64 * 64 + (wq >> 1) * 32;
                if (col0 < N) {
                    float v[32];
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] = stage_rows[rl * GEMM_EPI_STRIDE + (wq >> 1) * 32 + j];
                    epilogue_preload<MODE>(ep, M, N, row, col0, pre, lane, c64 == 0);
                    epilogue_chunk<MODE>(ep, M, N, row, col0, v, lane, pre);
                }
                ptx::bar_sync(1 + cw, 128);                     // the slab buffer is rewritten next
            }
            epilogue_finish<MODE>(ep, M, row, pre);
        }
    }
}

// ------------------------------------------------------------------ dispatch
template <int BLOCK_N, int MODE, int AMODE = 0, bool ASCALE = false>
static int launch_cfg(const CUtensorMap& ta, const CUtensorMap& tb, const pb200_gemm_epilogue& ep, int M, int N, int K,
                      cudaStream_t st, const ConvGeom* geom = nullptr) {
    using L = GemmSmem<BLOCK_N, ASCALE>;
    static DeviceOnce attr_set;
    if (attr_set.first()) {
        PB_CUDA(cudaFuncSetAttribute(gemm_f16_kernel<BLOCK_N, MODE, AMODE, ASCALE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     L::SMEM_BYTES));
    }
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    if (geom) g = *geom;
    CUtensorMap ts = ta;            // placeholder when unused
    if (ASCALE) {
        const int P = ep.rows_per_sample;
        const int ns = P >= GEMM_BLOCK_M ? 1 : GEMM_BLOCK_M / P;
        const int64_t samples = ((int64_t)M + P - 1) / P;
        PB_TRY(make_tmap_f16_2d_box(&ts, ep.a_scale, samples, K, ep.a_scale_ld, GEMM_BLOCK_K, ns, 0));
    }
    const int tiles_m = AMODE == 0 ? ceil_div(M, GEMM_BLOCK_M) : g.batch * g.tiles_y * g.tiles_x;
    const int n_units = tiles_m * ceil_div(N, BLOCK_N);
    const int grid = n_units < sm_count() ? n_units : sm_count();
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(GEMM_THREADS);
    cfg.dynamicSmemBytes = L::SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    static const bool pdl = getenv("PB200_NO_PDL") == nullptr;      // A/B knob
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    PB_CUDA(cudaLaunchKernelEx(&cfg, gemm_f16_kernel<BLOCK_N, MODE, AMODE, ASCALE>, ta, tb, ts, ep, g, M, N, K));
    PB_LAUNCH_CHECK();
    return 0;
}

// im2col-free convolution: A gathered from an NHWC fp16 activation (see ConvGeom); fp32 NHWC output (+bias)
int gemm_conv_launch(const CUtensorMap& ta, const CUtensorMap& tb, int block_n, const pb200_gemm_epilogue& ep,
                     const ConvGeom& geom, int64_t N, int64_t K, cudaStream_t st) {
    PB_CHECK(ep.mode == PB200_EPI_F32, "conv gemm: only the fp32 store epilogue is instantiated");
    PB_CHECK(geom.mode == 1 || geom.mode == 2, "conv gemm: bad mode");
    PB_CHECK(geom.tw * geom.th == GEMM_BLOCK_M, "conv gemm: tile must cover 128 positions");
    const int64_t M = (int64_t)geom.batch * geom.oh * geom.ow;     // rows of the output tensor (mask value in-kernel)
    PB_CHECK(M < (1ll << 31) && N % 8 == 0, "conv gemm: problem too large / N not a multiple of 8");
    ProfScope prof(geom.mode == 1 ? "conv_k4s2" : "convT_k4s2", 2.0 * (double)geom.batch * geom.gh * geom.gw * (double)N * (double)K, st);
#define PB_CONV_CASE(BN)                                                                                           \
    case BN:                                                                                                       \
        return geom.mode == 1 ? launch_cfg<BN, PB200_EPI_F32, 1>(ta, tb, ep, (int)M, (int)N, (int)K, st, &geom)    \
                              : launch_cfg<BN, PB200_EPI_F32, 2>(ta, tb, ep, (int)M, (int)N, (int)K, st, &geom);
    switch (block_n) {
        PB_CONV_CASE(64)
        PB_CONV_CASE(128)
        PB_CONV_CASE(256)
    }
#undef PB_CONV_CASE
    PB_CHECK(false, "conv gemm: unsupported BLOCK_N %d", block_n);
    return 1;
}

template <int BLOCK_N>
static int launch_mode(const CUtensorMap& ta, const CUtensorMap& tb, const pb200_gemm_epilogue& ep, int M, int N, int K,
                       cudaStream_t st) {
    if (ep.a_scale) {       // GlobalResponseNorm folded into the A operand: the two residual epilogues only
        if (ep.mode == PB200_EPI_RESID_F32) return launch_cfg<BLOCK_N, PB200_EPI_RESID_F32, 0, true>(ta, tb, ep, M, N, K, st);
        if (ep.mode == PB200_EPI_RESID_LN_F32) return launch_cfg<BLOCK_N, PB200_EPI_RESID_LN_F32, 0, true>(ta, tb, ep, M, N, K, st);
        PB_CHECK(false, "gemm: a_scale is only built for the RESID epilogues (mode %d)", ep.mode);
    }
    switch (ep.mode) {
        case PB200_EPI_F16: return launch_cfg<BLOCK_N, PB200_EPI_F16>(ta, tb, ep, M, N, K, st);
        case PB200_EPI_F32: return launch_cfg<BLOCK_N, PB200_EPI_F32>(ta, tb, ep, M, N, K, st);
        case PB200_EPI_GELU_F16: return launch_cfg<BLOCK_N, PB200_EPI_GELU_F16>(ta, tb, ep, M, N, K, st);
        case PB200_EPI_RESID_F32: return launch_cfg<BLOCK_N, PB200_EPI_RESID_F32>(ta, tb, ep, M, N, K, st);
        case PB200_EPI_UNPATCH_F32: return launch_cfg<BLOCK_N, PB200_EPI_UNPATCH_F32>(ta, tb, ep, M, N, K, st);
        case PB200_EPI_NCHW_F32: return launch_cfg<BLOCK_N, PB200_EPI_NCHW_F32>(ta, tb, ep, M, N, K, st);
        case PB200_EPI_RESID_LN_F32: return launch_cfg<BLOCK_N, PB200_EPI_RESID_LN_F32>(ta, tb, ep, M, N, K, st);
        case PB200_EPI_F16_LN: return launch_cfg<BLOCK_N, PB200_EPI_F16_LN>(ta, tb, ep, M, N, K, st);
    }
    PB_CHECK(false, "gemm: unknown epilogue mode %d", ep.mode);
    return 1;
}

// planning-only override of the multiprocessor count (pb200_gemm_plan); 0 = ask the device
static thread_local int g_plan_sms = 0;
static int plan_sm_count() {
    if (g_plan_sms > 0) return g_plan_sms;
    const int s = sm_count();
    return s > 0 ? s : 132;
}

bool gemm_can_scale_a(int64_t M, int64_t N, int64_t K, int rows_per_sample) {
    (void)M; (void)N;
    const int P = rows_per_sample;
    if (P <= 0 || K % GEMM_BLOCK_K != 0) return false;
    return P >= GEMM_BLOCK_M ? P % GEMM_BLOCK_M == 0 : (GEMM_BLOCK_M % P == 0 && GEMM_BLOCK_M / P <= 8);
}

int gemm_pick_block_n(int64_t M, int64_t N, int64_t K) {
    // Cycle model per candidate BLOCK_N, from the H100 SXM data sheet (not calibrated by measurement):
    //   tensor   : waves x k-blocks x 128 x BLOCK_N x 64 MACs at ~2048 fp16 MACs per clock and SM (989 TFLOP/s, 132 SMs)
    //   L2->SM   : all tiles' operand bytes (per k-block the 128x64 A tile and BLOCK_N x 64 of W) at ~3000 B/clk
    //   per tile : ~2000 cycles of fill/drain + the epilogue, which does not overlap the main loop
    // and pick the minimum.
    static const int force = getenv("PB200_FORCE_BN") ? atoi(getenv("PB200_FORCE_BN")) : 0;   // experiments only
    if (force == 64 || force == 128 || force == 256) return force;
    const int sms = plan_sm_count();
    const long n_kb = K > 0 ? (long)ceil_div(K, GEMM_BLOCK_K) : 16;
    const int cands[3] = {256, 128, 64};
    int best = 128;
    double best_cost = 1e30;
    for (int i = 0; i < 3; ++i) {
        const int bn = cands[i];
        const long units = (long)ceil_div(M, GEMM_BLOCK_M) * ceil_div(N, bn);
        const long waves = (units + sms - 1) / sms;
        const double mma = (double)waves * n_kb * 4.0 * bn;
        const double l2 = (double)units * n_kb * (16384.0 + bn * 128.0) / 3000.0;
        const double cost = (mma > l2 ? mma : l2) + waves * (2000.0 + 4.0 * bn);
        if (cost < best_cost) { best_cost = cost; best = bn; }
    }
    return best;
}

int gemm_launch(const CUtensorMap& ta, const CUtensorMap& tb, int block_n, const pb200_gemm_epilogue& ep, int64_t M,
                int64_t N, int64_t K, cudaStream_t st) {
    PB_CHECK(M > 0 && N > 0 && K > 0, "gemm: empty problem");
    PB_CHECK(N % 8 == 0, "gemm: N=%lld must be a multiple of 8", (long long)N);
    PB_CHECK(ep.out != nullptr, "gemm: null output");
    if (ep.mode == PB200_EPI_RESID_F32 || ep.mode == PB200_EPI_RESID_LN_F32)
        PB_CHECK(ep.resid != nullptr, "gemm: RESID epilogue without resid");
    if (ep.mode == PB200_EPI_RESID_LN_F32) PB_CHECK(ep.out16 && ep.ln_stat, "gemm: RESID_LN needs out16 and ln_stat");
    if (ep.mode == PB200_EPI_F16_LN)
        PB_CHECK(ep.ln_stat && ep.ln_wsum && ep.ln_c > 0, "gemm: F16_LN needs ln_stat, ln_wsum and ln_c");
    if (ep.mode == PB200_EPI_UNPATCH_F32)
        PB_CHECK(ep.up_cout % 8 == 0 && ep.up_cout * 4 == N && (int64_t)ep.up_h * ep.up_w > 0,
                 "gemm: bad un-patchify geometry");
    if ((ep.mode == PB200_EPI_GELU_F16 && ep.sqsum) || ((ep.mode == PB200_EPI_RESID_F32 || ep.mode == PB200_EPI_RESID_LN_F32) && ep.film) ||
        ep.mode == PB200_EPI_NCHW_F32)
        PB_CHECK(ep.rows_per_sample > 0, "gemm: rows_per_sample required");
    if (ep.a_scale)
        PB_CHECK(gemm_can_scale_a(M, N, K, ep.rows_per_sample) && ep.a_scale_ld % 8 == 0 && ((uintptr_t)ep.a_scale & 15) == 0,
                 "gemm: a_scale needs rows_per_sample dividing or divided by 128, K %% 64 == 0");
    static const char* kTags[8] = {"gemm_f16", "gemm_f32", "gemm_gelu_sqsum", "gemm_resid", "gemm_unpatch", "gemm_nchw",
                                   "gemm_resid", "gemm_f16"};
    ProfScope prof(ep.mode >= 0 && ep.mode < 8 ? kTags[ep.mode] : "gemm", 2.0 * (double)M * (double)N * (double)K, st);
    switch (block_n) {
        case 64: return launch_mode<64>(ta, tb, ep, (int)M, (int)N, (int)K, st);
        case 128: return launch_mode<128>(ta, tb, ep, (int)M, (int)N, (int)K, st);
        case 256: return launch_mode<256>(ta, tb, ep, (int)M, (int)N, (int)K, st);
    }
    PB_CHECK(false, "gemm: unsupported BLOCK_N %d", block_n);
    return 1;
}

int gemm_f16(const void* a, int64_t lda, const void* w, int64_t ldw, int64_t M, int64_t N, int64_t K,
             const pb200_gemm_epilogue& ep, cudaStream_t st) {
    PB_CHECK(K % 8 == 0, "gemm: K=%lld must be a multiple of 8", (long long)K);
    const int bn = gemm_pick_block_n(M, N, K);
    CUtensorMap ta, tb;
    PB_TRY(make_tmap_f16_2d(&ta, a, M, K, lda, GEMM_BLOCK_M));
    PB_TRY(make_tmap_f16_2d(&tb, w, N, K, ldw, bn / 2));      // W box = half a tile (see the producer)
    return gemm_launch(ta, tb, bn, ep, M, N, K, st);
}

}  // namespace pb

extern "C" int pb200_gemm_plan(int64_t m, int64_t n, int64_t k, int sm_count, int* block_n, int* two_sm, int* tail_block_n) {
    PB_CHECK(m > 0 && n > 0 && k > 0 && block_n && two_sm && tail_block_n, "gemm_plan: bad arguments");
    pb::g_plan_sms = sm_count > 0 ? sm_count : 0;
    const int bn = pb::gemm_pick_block_n(m, n, k);
    *block_n = bn;
    *two_sm = 0;            // Hopper has no 2-SM MMA: every tile is one CTA's
    *tail_block_n = 0;      // ... and every tile is BLOCK_N wide
    pb::g_plan_sms = 0;
    return 0;
}

extern "C" int pb200_gemm_f16(const void* a, int64_t lda, const void* w, int64_t ldw, int64_t m, int64_t n, int64_t k,
                              const pb200_gemm_epilogue* epi, void* stream) {
    PB_CHECK(epi != nullptr, "gemm: null epilogue");
    return pb::gemm_f16(a, lda, w, ldw, m, n, k, *epi, (cudaStream_t)stream);
}
