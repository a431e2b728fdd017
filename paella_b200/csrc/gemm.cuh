// Internal interface of the wgmma GEMM (see gemm.cu).
#pragma once
#include "common.cuh"
#include "paella_b200.h"
#include "ptx.cuh"

namespace pb {

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;     // 64 fp16 = one 128-byte swizzle row
constexpr int GEMM_CONSUMERS = 2;    // MMA warpgroups, 64 rows of the tile each
constexpr int GEMM_THREADS = 128 * (1 + GEMM_CONSUMERS);      // + the producer warpgroup
constexpr int GEMM_EPI_STRIDE = 65;  // fp32 row stride of the epilogue slab (odd: the row-per-lane reads are conflict-free)
constexpr int GEMM_EPI_BYTES = GEMM_CONSUMERS * 64 * GEMM_EPI_STRIDE * 4;
constexpr int SMEM_PER_BLOCK_MAX = 232448;     // 227 KB: the opt-in limit of one block on sm_90

template <int BLOCK_N>
struct GemmSmem {
    static constexpr int A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
    static constexpr int B_BYTES = BLOCK_N * GEMM_BLOCK_K * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int FIXED = GEMM_EPI_BYTES + 1024 /*alignment slack*/ + 256 /*barriers*/;
    static constexpr int FIT = (SMEM_PER_BLOCK_MAX - FIXED) / STAGE_BYTES;
    static constexpr int STAGES = FIT > 8 ? 8 : FIT;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED;
};

// 2-D fp16 tensor map over a row-major [rows, cols] matrix with leading dimension ld (elements):
// box = 64 columns x box_rows rows, 128-byte swizzle, zero fill out of bounds.
int make_tmap_f16_2d(CUtensorMap* tm, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows);

// same with an explicit box (box_cols x box_rows) and swizzle span (128 or 32 bytes; box_cols * 2 <= swizzle_bytes)
int make_tmap_f16_2d_box(CUtensorMap* tm, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows,
                         int swizzle_bytes);

// ... through a process-wide cache keyed by (pointer, shape, box, swizzle)
int cached_tmap_f16_2d(const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_cols, int box_rows, int swizzle_bytes,
                       CUtensorMap* out);

int make_tmap_f16_nd(CUtensorMap* tm, const void* ptr, int rank, const int64_t* dims, const int64_t* strides_bytes,
                     const int* box);

// A operand gathered from an NHWC fp16 activation instead of a matrix (im2col-free convolutions of the VQGAN):
//   mode 1  Conv2d(k=4,s=2,p=1):        5-D map over the [B, H/2, 2, W/2, 2*C] view, 16 taps
//   mode 2  ConvTranspose2d(k=4,s=2,p=1), one output phase (py,px): 4-D map [B,H,W,C], 4 taps
struct ConvGeom {
    int mode;
    int batch;
    int tw, th;               // a 128-row tile = th x tw positions of the GEMM-row grid
    int tiles_x, tiles_y;
    int gh, gw;               // GEMM-row grid (mode 1: conv output grid; mode 2: convT input grid)
    int cin, n_cchunk;        // input channels, ceil(cin / 64)
    int oh, ow, sy, sx, py, px;   // output pixel of grid position (y,x): ((b*oh + y*sy + py)*ow + x*sx + px)
    int org;                  // mode 2: map coordinate of grid position 0 (1 when the map covers a [B,H+2,W+2,C] bordered copy)
};

int gemm_conv_launch(const CUtensorMap& ta, const CUtensorMap& tb, int block_n, const pb200_gemm_epilogue& ep,
                     const ConvGeom& geom, int64_t N, int64_t K, cudaStream_t st);

// BLOCK_N that minimises a tensor / L2 cycle model of the launch (see gemm.cu)
int gemm_pick_block_n(int64_t M, int64_t N, int64_t K = 0);

// tb: tensor map of W with box rows block_n / 2
int gemm_launch(const CUtensorMap& ta, const CUtensorMap& tb, int block_n, const pb200_gemm_epilogue& ep, int64_t M,
                int64_t N, int64_t K, cudaStream_t st);

// convenience: builds both tensor maps and launches
int gemm_f16(const void* a, int64_t lda, const void* w, int64_t ldw, int64_t M, int64_t N, int64_t K,
             const pb200_gemm_epilogue& ep, cudaStream_t st);

// In-warp 8x8 transpose of float4 items (xor-butterfly shuffles): the epilogue hands lane l row l of a 32-column chunk; afterwards
// item i of lane (a, b) = row 8a + i, columns 4b..4b+3, so one store instruction writes four full 128-byte lines.
__device__ __forceinline__ void transpose8x8_f4(float (&v)[32], int lane) {
#pragma unroll
    for (int s = 4; s > 0; s >>= 1) {
        const bool up = (lane & s) != 0;
#pragma unroll
        for (int g0 = 0; g0 < 8; ++g0) {
            if (g0 & s) continue;
            const int g1 = g0 | s;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float send = up ? v[g0 * 4 + e] : v[g1 * 4 + e];
                const float recv = __shfl_xor_sync(0xffffffffu, send, s);
                if (up) v[g0 * 4 + e] = recv;
                else v[g1 * 4 + e] = recv;
            }
        }
    }
}

}  // namespace pb
