// Native unit test of AttentionKVCache's rolling-cache attribute (no GPU, no CUDA symbols): linked against core.o /
// operators.o / schedule.o only.  Built and run by tests/test_ring_host.py::test_native_attribute_vector.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "core.h"
#include "operators.h"

using namespace infini;

static int g_failed = 0;
#define CHECK(cond)                                                                   \
    do {                                                                              \
        if (!(cond)) {                                                                \
            std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond);               \
            ++g_failed;                                                               \
        }                                                                             \
    } while (0)

namespace {
class PlanRuntime final : public RuntimeObj {
  public:
    PlanRuntime() : RuntimeObj(Device::CPU, -1) {}
    void run(const Graph &, bool, bool) const override { throw Exception("no kernels on the host"); }
    void *alloc(size_t size) override { return std::aligned_alloc(256, ((std::max<size_t>(size, 1) + 255) / 256) * 256); }
    void dealloc(void *ptr) override { std::free(ptr); }
    void sync() const override {}
    void copyBlobFromCPU(void *d, const void *s, size_t n) const override { std::memcpy(d, s, n); }
    void copyBlobToCPU(void *d, const void *s, size_t n) const override { std::memcpy(d, s, n); }
    void copyBlobInsideRuntime(void *d, const void *s, size_t n) const override { std::memmove(d, s, n); }
    string toString() const override { return "native-test planning runtime"; }
};
}  // namespace

// a linear cache keeps the attribute vector of its window (or of no window); a ring appends 1 after the window
static Operator attention(Graph &g, bool perRow, int window, bool rolling) {
    const DataType bf = DataType::BFloat16;
    return g->addOp<AttentionKVCacheObj>(g->addTensor({2, 2, 64, 128}, bf), g->addTensor({2, 2, 64, 128}, bf),
                                         g->addTensor({2, 8, 1, 128}, bf), g->addTensor({2, 2, 1, 128}, bf),
                                         g->addTensor({2, 2, 1, 128}, bf), g->addTensor({2, 1}, DataType::Int64), nullptr, perRow,
                                         nullptr, nullptr, window, rolling);
}

int main() {
    Runtime rt = make_ref<PlanRuntime>();
    Graph g = make_ref<GraphObj>(rt);
    const int type = (int)OpType(OpType::AttentionKVCache).underlying();
    for (bool perRow : {false, true}) {
        CHECK((attention(g, perRow, 0, false)->getOpAttrVector() == vector<int>{type, (int)perRow}));
        CHECK((attention(g, perRow, 48, false)->getOpAttrVector() == vector<int>{type, (int)perRow, 48}));
        CHECK((attention(g, perRow, 48, true)->getOpAttrVector() == vector<int>{type, (int)perRow, 48, 1}));
    }
    if (g_failed) {
        std::printf("%d check(s) failed\n", g_failed);
        return 1;
    }
    std::printf("passed\n");
    return 0;
}
