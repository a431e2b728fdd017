// The log-probability of each drawn token under its sample's tempered logits, for confidence-guided renoising: the body of
// token_score_kernel (score_body.cuh) with LOGP = true.  Replaces log_softmax(logits / T) over the [rows, num_labels] logits
// the reference would materialise; 4 bytes per row here.
#include "../score_body.cuh"
#include "confidence.h"

namespace pb {

// logp_out[r] = log_softmax(l_r * (1/T))[targets[r]] with 1/T = params[3 (r / hw) + 2]
__global__ void __launch_bounds__(SC_THREADS, 1)
token_logprob_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w, int R, int NL, int Kc,
                     int hw, const float* __restrict__ params, const int64_t* __restrict__ targets, float* __restrict__ logp_out) {
    token_score_body<true>(&tm_a, &tm_w, R, NL, Kc, 0.f, hw, params, targets, logp_out, nullptr, nullptr);
}

}  // namespace pb

extern "C" cudaError_t pbc_token_logprob_launch(const CUtensorMap* tm_a, const CUtensorMap* tm_w, int R, int NL, int Kc, int hw,
                                                const float* params, const int64_t* targets, float* logp_out, cudaStream_t st) {
    using namespace pb;
    // a per-device property, and cheap: set on every call rather than cached per device
    cudaError_t e = cudaFuncSetAttribute(token_logprob_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SC_SMEM);
    if (e != cudaSuccess) return e;
    token_logprob_kernel<<<(unsigned)ceil_div(R, 128), SC_THREADS, SC_SMEM, st>>>(*tm_a, *tm_w, R, NL, Kc, hw, params, targets,
                                                                                 logp_out);
    return cudaGetLastError();
}
