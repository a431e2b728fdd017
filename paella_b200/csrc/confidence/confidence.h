// The device code of confidence-guided renoising, built into its own library (libpaella_b200_confidence.so, see the Makefile):
// the two kernels and one launcher each.  libpaella_b200.so validates the arguments, builds the tensor maps and Philox streams,
// and calls these; they return the launch's CUDA error.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../common.cuh"

extern "C" {
// token_logprob_kernel over R token rows (tm_a: the fp16 operand [R, Kc], 128-row boxes; tm_w: the out_mapper weight [NL, Kc],
// 128-label boxes): logp_out[r] = log_softmax(l_r * (1/T))[targets[r]], 1/T = params[3 (r / hw) + 2].  Kc <= 256.
cudaError_t pbc_token_logprob_launch(const CUtensorMap* tm_a, const CUtensorMap* tm_w, int R, int NL, int Kc, int hw,
                                     const float* params, const int64_t* targets, float* logp_out, cudaStream_t st);
// renoise_confidence_kernel, one CTA per sample (batch >= 1, 1 <= hw <= PBC_RENOISE_MAX_HW): see pb200_renoise_confidence.
// seed_off NULL: one stream s over batch * hw elements; else sample b on seed_off[b] with the stride of s.
cudaError_t pbc_renoise_confidence_launch(const int64_t* x, const int64_t* random_x, const int64_t* src, const uint8_t* region,
                                          const int* slot, const float* logp, const float* t, const float* tau, int64_t batch,
                                          int64_t hw, pb::TorchPhilox s, const uint64_t* seed_off, int64_t* out, int64_t* mask_out,
                                          cudaStream_t st);
}

#define PBC_RENOISE_MAX_HW 32768      // the selection keeps a sample's keys (4 bytes per token) in shared memory: 128 KB
