// Fused out_mapper + log-softmax statistics per token row (see score.cu).
#pragma once
#include "common.cuh"

namespace pb {
// a16: fp16 [R, Kc] features; w16: fp16 [NL, Kc] out_mapper weight; targets: int64 [R].  Writes per row nll = lse - l_y
// (NaN for a target outside [0, NL)), smooth = lse - mean_j l_j (fp32 [R] each) and the first arg-max (int64 [R]).
int launch_token_scores(const __half* a16, int64_t R, int Kc, const __half* w16, int NL, const int64_t* targets, float* nll_out,
                        float* smooth_out, int64_t* argmax_out, cudaStream_t st);
}  // namespace pb
