// Fused out_mapper + Gumbel-max draw (see sampler.cu).
#pragma once
#include "common.cuh"

namespace pb {
// rows the fp16 feature buffer must be able to hold for R token rows (whole 4*rs-row Philox blocks)
int64_t fused_sampler_rows_padded(int64_t R, int NL);
// a16: fp16 [R, Kc] guided features; w16: fp16 [NL, Kc] out_mapper weight; out: int64 [R]
int launch_fused_sampler(const __half* a16, int64_t R, int Kc, const __half* w16, int NL, float inv_t, uint64_t seed,
                         uint64_t offset, int64_t* out, cudaStream_t st);
// the same draw with one stream per sample: a16 fp16 [n_samp * hw, Kc] (holding (n_samp - 1) * hw +
// fused_sampler_rows_padded(hw, NL) rows), seed_off DEVICE uint64 [n_samp][2] = (seed, philox offset); out int64 [n_samp * hw]
int launch_fused_sampler_per_sample(const __half* a16, int64_t n_samp, int64_t hw, int Kc, const __half* w16, int NL,
                                    float inv_t, const uint64_t* seed_off, int64_t* out, cudaStream_t st);
// per-sample parameters: params DEVICE float [n_samp][3] = (cfg, 1 - cfg, 1/T) of each sample of hw rows (only 1/T is read
// here).  seed_off == nullptr: one stream (seed, offset) over all n_samp * hw rows, as launch_fused_sampler; otherwise one
// stream per sample, as launch_fused_sampler_per_sample.  params == nullptr: every row uses inv_t.
// skip (per-sample streams only): DEVICE int32 [n_samp]; a sample with skip[b] != 0 does not draw, its rows of out are not
// written (and its seed_off entry is not read).  nullptr: every sample draws.
// top_k / top_p (with params, both or neither): DEVICE int32 [n_samp] and float [n_samp], sample b's top-k and top-p (0 and
// 1.0 are off; see TruncSmem in sampler.cu); nullptr: the untruncated instances.
int launch_fused_sampler_params(const __half* a16, int64_t n_samp, int64_t hw, int Kc, const __half* w16, int NL, float inv_t,
                                const float* params, uint64_t seed, uint64_t offset, const uint64_t* seed_off, int64_t* out,
                                cudaStream_t st, const int* skip = nullptr, const int* top_k = nullptr,
                                const float* top_p = nullptr);
}  // namespace pb
