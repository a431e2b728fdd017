// Segmented LoRA shrink + expand on rows of a linear layer's input and output (see lora.cu).
#pragma once
#include "common.cuh"
#include "paella_b200.h"

namespace pb {

constexpr int LORA_MAX_RANK = 64;

// One adapter's operands for one target, as stored in its packed blob (paella_b200/lora.py):
//   a    fp16 [rank_pad][K]  (rows >= rank are zero)
//   b    fp16 [N][rank_pad]  (columns >= rank are zero)
//   aux  fp32 [rank_pad + 1]: the row sums of the fp16 A rows (folded LayerNorm input), then alpha / rank
struct LoraOperand {
    const __half* a;
    const __half* b;
    const float* aux;
    int rank_pad;         // multiple of 8, <= LORA_MAX_RANK; 0 = the adapter does not cover this target
};
struct LoraOperands {
    LoraOperand op[PB200_LORA_MAX_ADAPTERS];
};

// For rows m < M with id = row_adapter[m / rows_per_entry] >= 0 and s = row_scale[m / rows_per_entry] != 0:
//   u[j] = sum_k x[m, k] a_id[j, k]                       (plain), or
//   u[j] = rstd_m (sum_k x[m, k] a_id[j, k] - mean'_m rowsum_id[j])   (ln_stat != NULL: x = a16 = fp16(row - shift) and
//          (mean', rstd) from ln_stat [M][2] over K columns, as the PB200_EPI_F16_LN GEMM epilogue derives them)
//   y[o, n] += s * (alpha/rank)_id * sum_j u[j] b_id[n, j]   for n < N, o = (m / remap_in) * remap_out + m % remap_in
// y is fp16 (rounded once after the add) or fp32.  Every other row of x and y is neither read nor written.  Each row's result
// depends only on its own x row, adapter and scale: no split-K, no atomics, fixed summation order.  K % 8 == 0, ldx % 8 == 0,
// N and ldy even.  u_ws: scratch of M * PB200_LORA_WORKSPACE_PER_ROW bytes (u of each row).
int launch_lora(const __half* x, int64_t ldx, int64_t M, int K, int N, int rows_per_entry, const int* row_adapter,
                const float* row_scale, const LoraOperands& ops, const int64_t* ln_stat, void* y, int64_t ldy, bool y_f32,
                int remap_in, int remap_out, float* u_ws, cudaStream_t st);

}  // namespace pb
