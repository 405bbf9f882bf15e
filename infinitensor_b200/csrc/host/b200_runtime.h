// b200_runtime.h -- the B200 device runtime (Device::CUDA) behind RuntimeObj.
//
// API-compatible with the reference's CudaRuntimeObj (include/cuda/cuda_runtime.h:70-110,
// src/cuda/cuda_runtime.cc): run / runWithoutSync / runWithCudaGraph / tune / alloc / copyBlob* /
// initComm / getWorkspace, the CUDA-graph capture cache with LRU eviction and invalidation on
// topology / storage / shape change (cuda_runtime.cc:52-65,210-283,351-426), and the thread-local
// current stream (include/cuda/cuda_common.h:115-139).  What is deliberately absent: cudnn / cublas
// handles (cuda_runtime.cc:83-86) -- every kernel here is our own.
#pragma once
#include <cuda_runtime.h>

#include <list>
#include <mutex>
#include <unordered_map>

#include "core.h"

namespace infini {

#define checkCudaError(call)                                                                   \
    do {                                                                                       \
        cudaError_t err__ = (call);                                                            \
        if (err__ != cudaSuccess)                                                              \
            throw ::infini::Exception(string("CUDA error: ") + cudaGetErrorString(err__) + " at " + __FILE__ + \
                                      ":" + std::to_string(__LINE__));                         \
    } while (0)

class CUDAStream {
    static thread_local cudaStream_t current;

  public:
    static cudaStream_t getCurrentStream() { return current; }
    class Guard {
        cudaStream_t prev;

      public:
        explicit Guard(cudaStream_t s) : prev(current) { current = s; }
        ~Guard() { current = prev; }
    };
};

class CommunicatorObj {
  protected:
    int worldSize, rank;

  public:
    CommunicatorObj(int worldSize, int rank) : worldSize(worldSize), rank(rank) {}
    virtual ~CommunicatorObj() = default;
    int getWorldSize() const { return worldSize; }
    int getRank() const { return rank; }
    virtual void *getNcclComm() const = 0;
};
Ref<CommunicatorObj> makeNcclCommunicator(const string &name, int worldSize, int rank);
Ref<CommunicatorObj> makeNcclCommunicatorWithId(const void *id, int idBytes, int worldSize, int rank);
int ncclUniqueIdBytes(void *out, int outBytes);

class CudaRuntimeObj : public RuntimeObj {
    cudaStream_t stream = nullptr;
    mutable void *workspace = nullptr;
    mutable size_t workspaceSize = 0;
    // conv filters re-ordered for the implicit-GEMM kernel, one buffer per weight tensor (keyed by its device address), refilled at
    // the start of every step by ONE batched launch (b200::prepConvFilters) -- never a stale copy of weights the user has rewritten
    mutable std::unordered_map<const void *, std::pair<void *, size_t>> packedFilters;
    Ref<CommunicatorObj> comm;
    void *p2pLocal = nullptr;
    void *p2pWs[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    int p2pWorld = 0, p2pRankId = 0;
    int *p2pTimeoutHost = nullptr, *p2pTimeoutDev = nullptr;  // host-mapped flag the all-reduce kernel raises when a peer never arrives
    void checkPeerTimeout() const;
    mutable std::recursive_mutex executionMutex;

    struct TensorSig {
        void *ptr;
        Shape dims;
        int dtype;
        bool operator==(const TensorSig &o) const { return ptr == o.ptr && dims == o.dims && dtype == o.dtype; }
    };
    struct CacheEntry {
        uint64_t graphId, topologyEpoch, storageEpoch;
        vector<TensorSig> sig;
        cudaGraphExec_t exec = nullptr;
        cudaGraph_t graph = nullptr;
    };
    mutable std::list<CacheEntry> cache;  // front = most recently used
    size_t cacheCapacity;
    mutable size_t captureCount = 0;
    mutable bool capturing = false;

    // per-(graph, topology epoch) dispatch plan: kernel pointers + perf keys resolved once
    struct PlanEntry {
        Kernel *kernel;  // kernel of the step's LAST operator (the only one used by Single / Alias steps)
        std::optional<PerfRecord> record;
    };
    mutable uint64_t planGraphId = 0, planEpoch = ~0ull;
    mutable vector<PlanEntry> plan;

    void runWithoutSyncImpl(const Graph &graph, bool validate) const;
    void execStep(const ExecStep &st, Kernel *kernel, const PerfRecord *record) const;
    vector<TensorSig> signature(const Graph &graph) const;
    void destroyEntry(CacheEntry &e) const;
    void recoverStream() const;
    void tune(const Graph &graph) const;

  public:
    explicit CudaRuntimeObj(int deviceId = 0, size_t cudaGraphCacheCapacity = 16);
    ~CudaRuntimeObj() override;
    string toString() const override { return "B200 CUDA Runtime (device " + std::to_string(deviceId) + ")"; }

    void run(const Graph &graph, bool tune = false, bool profiling = false) const override;
    void runWithoutSync(const Graph &graph) const;
    void runWithCudaGraph(const Graph &graph, bool syncAfter = true) const;
    void sync() const override;

    void *alloc(size_t size) override;
    void dealloc(void *ptr) override;
    void copyBlobFromCPU(void *dst, const void *src, size_t bytes) const override;
    void copyBlobToCPU(void *dst, const void *src, size_t bytes) const override;
    void copyBlobInsideRuntime(void *dst, const void *src, size_t bytes) const override;
    // stream-ordered variants (pinned host memory) used by the serving loop
    void copyBlobFromCPUAsync(void *dst, const void *src, size_t bytes) const;
    void copyBlobToCPUAsync(void *dst, const void *src, size_t bytes) const;

    // one scratch buffer, always the same base pointer (reference cuda_runtime.h:85-88)
    void *getWorkspace(size_t size) const;
    size_t getWorkspaceSize() const { return workspaceSize; }
    void *packedFilterBuffer(const void *weights, size_t bytes) const;  // allocates on first use (outside CUDA-graph capture)
    std::pair<void *, size_t> findPackedFilter(const void *weights) const {
        auto it = packedFilters.find(weights);
        return it == packedFilters.end() ? std::pair<void *, size_t>{nullptr, 0} : it->second;
    }
    cudaStream_t getStream() const { return stream; }

    // NVLink peer-memory communicator for the fused one-shot all-reduce (kernels/allreduce.cu)
    void p2pExport(void *handle64);                                      // allocates the local comm workspace
    void p2pImport(const void *allHandles, int worldSize, int rank);     // maps every peer's workspace
    bool hasPeerComm() const { return p2pWorld > 0; }
    void *const *peerWorkspaces() const { return p2pWs; }
    int p2pWorldSize() const { return p2pWorld; }
    int p2pRank() const { return p2pRankId; }
    int *p2pTimeoutFlagDevice() const { return p2pTimeoutDev; }
    void initComm(const string &name, int worldSize, int rank);
    void initCommWithId(const void *id, int idBytes, int worldSize, int rank);
    CommunicatorObj &getCommunicator() const {
        IT_ASSERT(comm != nullptr, "communicator not initialised (call init_comm)");
        return *comm;
    }
    bool hasCommunicator() const { return comm != nullptr; }

    void clearCudaGraphCache() const;
    size_t getCudaGraphCacheSize() const { return cache.size(); }
    size_t getCudaGraphCaptureCount() const { return captureCount; }
    bool isCapturing() const { return capturing; }
};

// fused executors behind the ExecStep kinds (b200_kernels.cc)
namespace b200 {
void runMatmul(const Operator &op, const RuntimeObj *ctx, const Tensor &residual, const Tensor &outOverride);
void runMatmulGroup(const OpVec &ops, const RuntimeObj *ctx);
void runSiluMul(const Operator &silu, const Operator &mul, const RuntimeObj *ctx);
// AllReduceSum -> Add(residual) [-> RMSNorm]: true if the fused NVLink kernel took it, false = run the ops one by one
bool runAllReduceAddNorm(const OpVec &ops, const RuntimeObj *ctx);
// Conv -> BatchNorm -> [Add] -> [Relu] in the GEMM epilogue; false = shape not taken (nothing launched)
bool matmulAddIsPlain(const OpVec &ops);  // {bias-free MatMul, Add}: the residual rides the GEMM's bias slot (every GEMM kernel)
bool runMatmulFused(const OpVec &ops, const RuntimeObj *ctx);
bool runConvBnAct(const OpVec &ops, const RuntimeObj *ctx, int layout = 0);
void prepConvFilters(const vector<ExecStep> &sched, const RuntimeObj *ctx);
void runPoolNhwc(const Operator &op, const RuntimeObj *ctx);
void runAttentionRope(const Operator &ropeQ, const Operator &ropeK, const Operator &att, const RuntimeObj *ctx);
// {Transpose(k), MatMul, [Div | Mul], [Add], Softmax, MatMul} as one fused wgmma attention kernel
void runPrefillAttention(const OpVec &ops, const RuntimeObj *ctx);
}  // namespace b200

// Convenience base for kernels without tunable configs (reference cuda_kernel_wihtout_config.h:7-22)
class CudaKernelWithoutConfig : public Kernel {
  public:
    void compute(const Operator &op, const PerfRecord &, const RuntimeObj *context) const override {
        compute(op, context);
    }
    void compute(const Operator &op, const RuntimeObj *context) const override = 0;
    PerfRecord tune(const Operator &op, const RuntimeObj *context) const override;
};

}  // namespace infini
