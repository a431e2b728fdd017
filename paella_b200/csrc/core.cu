// Error plumbing, device queries and the measurement hooks shared by the whole library.
#include "common.cuh"
#include "paella_b200.h"

#include <nvtx3/nvToolsExt.h>     // header-only NVTX v3: ranges cost ~nothing unless a tool (nsys / ncu --nvtx) is attached

#include <atomic>
#include <cstring>
#include <map>
#include <mutex>
#include <sstream>
#include <vector>

namespace pb {

static thread_local std::string g_err;

void set_error(const std::string& msg) { g_err = msg; }
const char* last_error() { return g_err.c_str(); }

// per-device caches (a process may drive several GPUs: Paella on cuda:0, VQModel on cuda:1)
constexpr int kMaxDev = 64;
static int g_sm[kMaxDev], g_tpsm[kMaxDev];
static bool g_dev_known[kMaxDev];
static std::mutex g_dev_mu;
static int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); return -1; }
    return dev;
}
static int query_device() {
    const int dev = current_device();
    if (dev < 0 || dev >= kMaxDev) return -1;
    std::lock_guard<std::mutex> lk(g_dev_mu);
    if (!g_dev_known[dev]) {
        int sm = 0, tpsm = 2048;
        if (cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&tpsm, cudaDevAttrMaxThreadsPerMultiProcessor, dev) != cudaSuccess) {
            (void)cudaGetLastError();
            sm = 0; tpsm = 2048;
        }
        g_sm[dev] = sm; g_tpsm[dev] = tpsm; g_dev_known[dev] = true;
    }
    return dev;
}
int sm_count() { const int d = query_device(); return d < 0 ? 0 : g_sm[d]; }
int max_threads_per_sm() { const int d = query_device(); return d < 0 ? 2048 : g_tpsm[d]; }

bool DeviceOnce::first() {
    const int dev = current_device();
    if (dev < 0 || dev >= kMaxDev) return true;
    std::lock_guard<std::mutex> lk(g_dev_mu);
    const unsigned long long bit = 1ull << dev;
    if (mask & bit) return false;
    mask |= bit;
    return true;
}

// ------------------------------------------------------------------ measurement hooks
static std::atomic<long long> g_launches{0};
static bool g_prof = false;
struct ProfRec {
    std::string tag;
    double work;
    cudaEvent_t e0, e1;
};
static std::vector<ProfRec> g_recs;
static std::mutex g_prof_mu;

void prof_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
bool prof_enabled() { return g_prof; }

// Every kernel family launched by the library sits inside an NVTX range named after it ("gemm_gelu", "attention",
// "dwconv_ln", "fused_sampler", "vq_nearest", ...): `ncu --nvtx --nvtx-include "attention/"` or an nsys timeline can
// select a family without knowing mangled kernel names.
ProfScope::ProfScope(const char* tag, double work, cudaStream_t s) : slot(-1), st(s) {
    nvtxRangePushA(tag);
    if (!g_prof) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    ProfRec r;
    r.tag = tag;
    r.work = work;
    if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
    cudaEventRecord(r.e0, st);
    slot = (int)g_recs.size();
    g_recs.push_back(r);
}
ProfScope::~ProfScope() {
    nvtxRangePop();
    if (slot < 0) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    cudaEventRecord(g_recs[slot].e1, st);
}

}  // namespace pb

extern "C" {
const char* pb200_last_error(void) { return pb::last_error(); }
int pb200_abi_version(void) { return PB200_ABI_VERSION; }
int pb200_device_info(int* sms, int* tpsm) {
    PB_CHECK(pb::sm_count() > 0, "no CUDA device");
    if (sms) *sms = pb::sm_count();
    if (tpsm) *tpsm = pb::max_threads_per_sm();
    return 0;
}

long long pb200_launch_count(void) { return pb::g_launches.load(); }

int pb200_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(pb::g_prof_mu);
    for (auto& r : pb::g_recs) {
        cudaEventDestroy(r.e0);
        cudaEventDestroy(r.e1);
    }
    pb::g_recs.clear();
    pb::g_prof = on != 0;
    return 0;
}

// Synchronises the device and writes a JSON object {tag: {"launches": n, "ms": total, "work": total}} into buf.
int pb200_profile_report(char* buf, long long cap) {
    PB_CUDA(cudaDeviceSynchronize());
    std::lock_guard<std::mutex> lk(pb::g_prof_mu);
    struct Agg { long long n = 0; double ms = 0, work = 0; };
    std::map<std::string, Agg> agg;
    for (auto& r : pb::g_recs) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.e0, r.e1) != cudaSuccess) continue;
        Agg& a = agg[r.tag];
        a.n += 1; a.ms += ms; a.work += r.work;
    }
    std::ostringstream os;
    os.precision(9);
    os << "{";
    bool first = true;
    for (auto& kv : agg) {
        if (!first) os << ", ";
        first = false;
        os << "\"" << kv.first << "\": {\"launches\": " << kv.second.n << ", \"ms\": " << kv.second.ms << ", \"work\": "
           << kv.second.work << "}";
    }
    os << "}";
    const std::string s = os.str();
    PB_CHECK((long long)s.size() + 1 <= cap, "profile_report: buffer too small");
    memcpy(buf, s.c_str(), s.size() + 1);
    return 0;
}
}
