// support.cu -- error string + launch counter shared by every launcher.
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
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
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
