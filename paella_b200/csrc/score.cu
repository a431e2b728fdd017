// Fused out_mapper GEMM + log-softmax statistics: per token row the negative log-likelihood of a target code, the
// label-smoothing term and the arg-max, without the logits ever reaching HBM.
// Replaces ref/utils/modules.py:268-280 (the out_mapper of Paella.forward) followed by src/train.py:64,71
// (nn.CrossEntropyLoss(label_smoothing, reduction='none') and pred.argmax(1)): [rows, num_labels] fp32 logits and their
// log_softmax in the reference, 16 bytes per row here.
//
// For row r with logits l = a16[r] . W^T (fp16 operands, fp32 accumulation) and target y = targets[r]:
//     lse    = log sum_j exp(l_j)
//     nll    = lse - l_y                      (NaN for y outside [0, NL): the target is compared, never used as an index)
//     smooth = lse - (1/NL) sum_j l_j         (CrossEntropyLoss's label-smoothing term: -mean_j log p_j)
//     argmax = the lowest j with l_j = max l (torch's tie rule)
//
// The layout is the fused sampler's generic one (sampler.cu): one CTA per 128 token rows, 384 threads,
//   warpgroup 0     TMA: the 128 x c_out A tile once (resident), then W tiles [128 labels x 64] through a 6-deep ring
//   warpgroups 1,2  wgmma m64n128k16 for 64 token rows each; per label chunk an online max and rescaled sum of exp, sum l,
//                   the running arg-max and l_y for each of the thread's two rows.  The quad of threads sharing a row is
//                   combined at the end in a fixed shuffle order, so a row's results depend only on its own A row.
#include "score_body.cuh"

namespace pb {

__global__ void __launch_bounds__(SC_THREADS, 1)
token_score_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w, int R, int NL, int Kc,
                   float inv_nl, const int64_t* __restrict__ targets, float* __restrict__ nll_out, float* __restrict__ smooth_out,
                   int64_t* __restrict__ argmax_out) {
    token_score_body<false>(&tm_a, &tm_w, R, NL, Kc, inv_nl, 1, nullptr, targets, nll_out, smooth_out, argmax_out);
}

int launch_token_scores(const __half* a16, int64_t R, int Kc, const __half* w16, int NL, const int64_t* targets, float* nll_out,
                        float* smooth_out, int64_t* argmax_out, cudaStream_t st) {
    PB_CHECK(Kc % 8 == 0 && Kc <= 64 * SC_MAX_KB, "token scores: c_out=%d unsupported (<= %d, multiple of 8)", Kc, 64 * SC_MAX_KB);
    PB_CHECK(NL > 0 && R >= 0 && R < (1ll << 31), "token scores: %lld rows of %d labels", (long long)R, NL);
    if (R == 0) return 0;
    static DeviceOnce attr_set;
    if (attr_set.first())
        PB_CUDA(cudaFuncSetAttribute(token_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SC_SMEM));
    ProfScope prof("token_scores", 2.0 * (double)R * (double)NL * (double)Kc, st);
    CUtensorMap ta, tw;
    PB_TRY(make_tmap_f16_2d(&ta, a16, R, Kc, Kc, 128));
    PB_TRY(make_tmap_f16_2d(&tw, w16, NL, Kc, Kc, SC_BN));
    token_score_kernel<<<(unsigned)ceil_div(R, 128), SC_THREADS, SC_SMEM, st>>>(ta, tw, (int)R, NL, Kc, 1.0f / (float)NL, targets,
                                                                               nll_out, smooth_out, argmax_out);
    PB_LAUNCH_CHECK();
    return 0;
}

}  // namespace pb
