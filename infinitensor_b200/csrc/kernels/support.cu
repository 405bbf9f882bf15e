// support.cu -- error string, launch counter and shared-memory opt-ins shared by every launcher.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>

#include "common.cuh"

namespace itb {
static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int launched(const char *what, cudaError_t e) {
    if (e != cudaSuccess) ITB_FAIL("%s: %s", what, cudaGetErrorString(e));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return 0;
}
// the attribute belongs to a (device, kernel) pair: a process may own runtimes on several GPUs, and every instance of a
// kernel template is its own kernel
int opt_in_smem(const char *what, const void *kernel, int smem) {
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, int> granted;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(mu);
    int &have = granted[{dev, kernel}];
    if (smem <= have) return 0;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) ITB_FAIL("%s: smem attribute: %s", what, cudaGetErrorString(e));
    have = smem;
    return 0;
}
bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char *e = std::getenv("ITB_NO_PDL");
        v = (e && e[0] == '1') ? 0 : 1;
    }
    return v == 1;
}
int *stream_tickets(cudaStream_t st, int n) {
    static std::mutex mu;
    static std::map<std::pair<int, cudaStream_t>, int *> table;
    constexpr int kPool = 65536;
    if (n > kPool) return nullptr;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(mu);
    int *&p = table[{dev, st}];
    if (!p) {
        if (cudaMalloc(&p, kPool * sizeof(int)) != cudaSuccess) return p = nullptr;
        if (cudaMemset(p, 0, kPool * sizeof(int)) != cudaSuccess) return nullptr;
    }
    return p;
}
long long launches() { return g_launches.load(std::memory_order_relaxed); }
}  // namespace itb

extern "C" const char *it_b200_last_error(void) { return itb::g_err; }
extern "C" int it_b200_version(void) { return 1; }
extern "C" long long it_b200_launch_count(void) { return itb::launches(); }
