// Shared device/host helpers for the paella_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace pb {

// ---------------------------------------------------------------- error plumbing
void set_error(const std::string& msg);
const char* last_error();

#define PB_CHECK(cond, ...)                                                             \
    do {                                                                                \
        if (!(cond)) {                                                                  \
            char _b[512];                                                               \
            snprintf(_b, sizeof(_b), __VA_ARGS__);                                      \
            pb::set_error(std::string(__FILE__) + ":" + std::to_string(__LINE__) + ": " + _b); \
            return 1;                                                                   \
        }                                                                               \
    } while (0)

#define PB_CUDA(expr)                                                                   \
    do {                                                                                \
        cudaError_t _e = (expr);                                                        \
        if (_e != cudaSuccess) {                                                        \
            pb::set_error(std::string(__FILE__) + ":" + std::to_string(__LINE__) + ": " + #expr + ": " + \
                          cudaGetErrorString(_e));                                      \
            return 1;                                                                   \
        }                                                                               \
    } while (0)

#define PB_LAUNCH_CHECK()            \
    do {                             \
        pb::prof_count_launch();     \
        PB_CUDA(cudaGetLastError()); \
    } while (0)

#define PB_TRY(expr)                 \
    do {                             \
        int _r = (expr);             \
        if (_r) return _r;           \
    } while (0)

inline int ceil_div(long a, long b) { return (int)((a + b - 1) / b); }

int sm_count();        // multiprocessor count of the CURRENT device (cached per device)
int max_threads_per_sm();
// One-time per-DEVICE setup (cudaFuncSetAttribute is a per-device property): true the first time it is called with this
// flag word while device d is current.  `static DeviceOnce once; if (once.first()) { ... }`
struct DeviceOnce {
    unsigned long long mask = 0;      // guarded by a library-wide mutex in first()
    bool first();
};

// ---------------------------------------------------------------- measurement hooks (bench.py)
void prof_count_launch();            // every kernel launch of the library bumps one counter
bool prof_enabled();
// When profiling is on, brackets the launches made in its scope with CUDA events on `st`, tagged with a kernel
// family and its algorithmic work (FLOPs for GEMM-shaped kernels, bytes otherwise).
struct ProfScope {
    int slot;
    cudaStream_t st;
    ProfScope(const char* tag, double work, cudaStream_t s);
    ~ProfScope();
};

// ---------------------------------------------------------------- small device helpers
// Lets a dependent kernel launched with programmatic stream serialization (the wgmma GEMMs, see ptx.cuh) start its
// prologue while this kernel's last CTAs are still running.  No effect otherwise.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// (-mean, rstd) of a row from the folded LayerNorm's fixed-point row statistics st = (sum x * 2^20, sum x^2 * 2^16) over c columns
// (PB200_EPI_RESID_LN*): the PB200_EPI_F16_LN epilogue and the LoRA shrink's fold both normalise with exactly these values
__device__ __forceinline__ void ln_stat_moments(const int64_t* st_row, int c, float& neg_mean, float& rstd) {
    const longlong2 st = *reinterpret_cast<const longlong2*>(st_row);
    const float inv_c = 1.0f / (float)c;
    const float mean = (float)st.x * (1.0f / 1048576.0f) * inv_c;
    const float ex2 = (float)st.y * (1.0f / 65536.0f) * inv_c;
    neg_mean = -mean;
    rstd = 1.0f / sqrtf(fmaxf(ex2 - mean * mean, 0.f) + 1e-6f);
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// Exact-erf GELU for the GEMM epilogue: erfc by Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, far below the fp16
// rounding of the stored activation), one MUFU.RCP + one MUFU.EX2 instead of libdevice erff's branches.  Written as
//   gelu(x) = max(x, 0) - |x| * u(|x|),   u(a) = 0.5 * erfc(a / sqrt2) = t * q(t) * exp(-a^2 / 2),  t = 1 / (1 + p a / sqrt2)
// (for x >= 0: x (1 - u); for x < 0: x u = -|x| u) with the 0.5 and 1/sqrt2 folded into the constants: 13 instructions
// per element -- the epilogue of the K=640 level is bound by instruction issue, not by the tensor pipe.
__device__ __forceinline__ float gelu_erf_fast(float x) {
    const float a = fabsf(x);
    float t, e;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752440f, a, 1.0f)));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"((x * x) * (-0.5f * 1.4426950408889634f)));     // exp(-x^2/2)
    float q = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);
    q = fmaf(q, t, 0.5f * 1.421413741f);
    q = fmaf(q, t, 0.5f * -0.284496736f);
    q = fmaf(q, t, 0.5f * 0.254829592f);
    return fmaf(-a, (q * t) * e, fmaxf(x, 0.f));
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- Philox4x32-10 (curand_philox4x32_x.h constants)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

// PyTorch's CUDA generator stream (ATen/native/cuda/DistributionTemplates.h:65-89): element e of a
// distribution kernel over `numel` elements is produced by thread tid = e % stride on its
// (e / stride / 4)-th curand4 call, lane (e / stride) % 4, where stride = 256 * grid.
struct TorchPhilox {
    uint64_t seed;
    uint64_t offset4;   // philox offset / 4 (PyTorch offsets are multiples of 4)
    uint32_t stride;    // 256 * grid
};

__device__ __forceinline__ uint4 torch_philox_call(const TorchPhilox& s, uint64_t tid, uint64_t call) {
    const uint64_t ctr = s.offset4 + call;
    return philox4x32_10(make_uint4((uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)tid, (uint32_t)(tid >> 32)),
                         make_uint2((uint32_t)s.seed, (uint32_t)(s.seed >> 32)));
}

__device__ __forceinline__ uint32_t torch_philox_u32(const TorchPhilox& s, uint64_t e) {
    const uint64_t j = e / s.stride;
    const uint64_t tid = e - j * s.stride;
    const uint4 r = torch_philox_call(s, tid, j >> 2);
    const uint32_t lane = (uint32_t)(j & 3);
    return lane == 0 ? r.x : lane == 1 ? r.y : lane == 2 ? r.z : r.w;
}

// curand_uniform: (0,1]
__device__ __forceinline__ float u32_to_uniform(uint32_t x) {
    return fmaf((float)x, 2.3283064365386963e-10f, 2.3283064365386963e-10f / 2.0f);
}

// Tensor.exponential_(1) CUDA branch (ATen/core/TransformationHelper.h:129-146): -log(u), with
// log(u) replaced by -eps/2 when u >= 1 - eps/2.  `at::log` on the device is the fast __logf
// (ATen/NumericUtils.h:149-160); using logf() here flips ~1e-4 of the draws.
__device__ __forceinline__ float torch_exponential1(float u) {
    const float lg = (u >= 1.0f - 1.1920928955078125e-07f / 2.0f) ? -(1.1920928955078125e-07f / 2.0f) : __logf(u);
    return -1.0f * lg;
}

TorchPhilox make_torch_philox(uint64_t seed, uint64_t offset, long numel);   // host: launch-policy stride for `numel`

}  // namespace pb
