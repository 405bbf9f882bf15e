// b200_runtime.cc -- see b200_runtime.h.  Run loop, CUDA-graph capture cache, memory, workspace.
#include "b200_runtime.h"

#include "it_b200.h"

#include <nvtx3/nvToolsExt.h>  // header-only; the ranges cost nothing unless a profiler is attached AND ITB_NVTX=1

#include <algorithm>
#include <cstdlib>

namespace infini {

thread_local cudaStream_t CUDAStream::current = nullptr;

CudaRuntimeObj::CudaRuntimeObj(int deviceId, size_t cudaGraphCacheCapacity)
    : RuntimeObj(Device::CUDA, deviceId), cacheCapacity(cudaGraphCacheCapacity) {
    checkCudaError(cudaSetDevice(deviceId));
    checkCudaError(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
}

CudaRuntimeObj::~CudaRuntimeObj() {
    cudaSetDevice(deviceId);
    if (stream) cudaStreamSynchronize(stream);
    for (auto &e : cache) destroyEntry(e);
    cache.clear();
    comm.reset();
    for (int p = 0; p < p2pWorld; ++p)
        if (p != p2pRankId && p2pWs[p]) cudaIpcCloseMemHandle(p2pWs[p]);
    if (p2pLocal) cudaFree(p2pLocal);
    if (p2pTimeoutHost) cudaFreeHost(p2pTimeoutHost);
    if (workspace) cudaFree(workspace);
    for (auto &kv : packedFilters) cudaFree(kv.second.first);
    if (stream) cudaStreamDestroy(stream);
}

void *CudaRuntimeObj::packedFilterBuffer(const void *weights, size_t bytes) const {
    auto it = packedFilters.find(weights);
    if (it != packedFilters.end() && it->second.second >= bytes) return it->second.first;
    IT_ASSERT(!capturing, "conv filter buffer requested during CUDA-graph capture (the eager pass before it allocates them)");
    if (it != packedFilters.end()) {
        checkCudaError(cudaStreamSynchronize(stream));
        cudaFree(it->second.first);
        packedFilters.erase(it);
    }
    void *p = nullptr;
    checkCudaError(cudaMalloc(&p, bytes));
    packedFilters[weights] = {p, bytes};
    return p;
}

void *CudaRuntimeObj::alloc(size_t size) {
    checkCudaError(cudaSetDevice(deviceId));
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, std::max<size_t>(size, 1));
    if (e != cudaSuccess) {
        cudaGetLastError();
        throw std::bad_alloc();
    }
    return p;
}
void CudaRuntimeObj::dealloc(void *ptr) {
    cudaSetDevice(deviceId);
    cudaFree(ptr);
}
void CudaRuntimeObj::sync() const {
    checkCudaError(cudaStreamSynchronize(stream));
    checkPeerTimeout();
}
// the peer-memory all-reduce gave up waiting for a rank (allreduce.cu): surfaced here, after the step, as a recoverable error
void CudaRuntimeObj::checkPeerTimeout() const {
    if (!p2pTimeoutHost) return;
    int v = *(volatile int *)p2pTimeoutHost;
    if (v == 0) return;
    *(volatile int *)p2pTimeoutHost = 0;
    int code = v - 1;
    throw Exception("peer-memory all-reduce timed out: rank " + std::to_string(code / 16) + " never received the packets of rank " +
                    std::to_string(code % 16) + " (dead or stalled peer); the step's outputs are invalid");
}

void CudaRuntimeObj::copyBlobFromCPU(void *dst, const void *src, size_t bytes) const {
    checkCudaError(cudaSetDevice(deviceId));
    checkCudaError(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
    checkCudaError(cudaStreamSynchronize(stream));
}
void CudaRuntimeObj::copyBlobToCPU(void *dst, const void *src, size_t bytes) const {
    checkCudaError(cudaSetDevice(deviceId));
    checkCudaError(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, stream));
    checkCudaError(cudaStreamSynchronize(stream));
}
void CudaRuntimeObj::copyBlobInsideRuntime(void *dst, const void *src, size_t bytes) const {
    checkCudaError(cudaSetDevice(deviceId));
    checkCudaError(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, stream));
    checkCudaError(cudaStreamSynchronize(stream));
}
void CudaRuntimeObj::copyBlobFromCPUAsync(void *dst, const void *src, size_t bytes) const {
    checkCudaError(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
}
void CudaRuntimeObj::copyBlobToCPUAsync(void *dst, const void *src, size_t bytes) const {
    checkCudaError(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, stream));
}

void *CudaRuntimeObj::getWorkspace(size_t size) const {
    if (size <= workspaceSize && workspace) return workspace;
    // grow (never while a capture is in flight: allocation is not capturable)
    IT_ASSERT(!capturing, "workspace must be sized before CUDA-graph capture (run the graph once eagerly)");
    size_t want = std::max<size_t>(size, 256ull << 20);
    if (const char *env = std::getenv("ITB_WORKSPACE_BYTES")) want = std::max<size_t>(want, strtoull(env, nullptr, 10));
    checkCudaError(cudaStreamSynchronize(stream));
    if (workspace) checkCudaError(cudaFree(workspace));
    workspace = nullptr;
    workspaceSize = 0;
    checkCudaError(cudaMalloc(&workspace, want));
    workspaceSize = want;
    // a new base pointer invalidates captured graphs that baked the old one in
    for (auto &e : cache) destroyEntry(e);
    cache.clear();
    return workspace;
}

void CudaRuntimeObj::p2pExport(void *handle64) {
    checkCudaError(cudaSetDevice(deviceId));
    if (!p2pLocal) {
        size_t bytes = (size_t)it_b200_allreduce_workspace_bytes();
        checkCudaError(cudaMalloc(&p2pLocal, bytes));
        checkCudaError(cudaMemset(p2pLocal, 0, bytes));
        checkCudaError(cudaDeviceSynchronize());
        checkCudaError(cudaHostAlloc((void **)&p2pTimeoutHost, sizeof(int), cudaHostAllocMapped));
        *p2pTimeoutHost = 0;
        checkCudaError(cudaHostGetDevicePointer((void **)&p2pTimeoutDev, p2pTimeoutHost, 0));
    }
    cudaIpcMemHandle_t h;
    checkCudaError(cudaIpcGetMemHandle(&h, p2pLocal));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    std::memcpy(handle64, &h, 64);
}
void CudaRuntimeObj::p2pImport(const void *allHandles, int worldSize, int rank) {
    IT_ASSERT(worldSize >= 1 && worldSize <= 8 && rank >= 0 && rank < worldSize, "p2p: bad world size / rank");
    IT_ASSERT(p2pLocal != nullptr, "p2p: export the local handle first");
    checkCudaError(cudaSetDevice(deviceId));
    for (int p = 0; p < worldSize; ++p) {
        if (p == rank) {
            p2pWs[p] = p2pLocal;
            continue;
        }
        cudaIpcMemHandle_t h;
        std::memcpy(&h, (const char *)allHandles + (size_t)p * 64, 64);
        void *ptr = nullptr;
        checkCudaError(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
        p2pWs[p] = ptr;
    }
    p2pWorld = worldSize;
    p2pRankId = rank;
}

void CudaRuntimeObj::initComm(const string &name, int worldSize, int rank) {
    IT_ASSERT(worldSize > 0 && rank >= 0 && rank < worldSize, "bad world size / rank");
    checkCudaError(cudaSetDevice(deviceId));
    comm = makeNcclCommunicator(name, worldSize, rank);
}
void CudaRuntimeObj::initCommWithId(const void *id, int idBytes, int worldSize, int rank) {
    IT_ASSERT(worldSize > 0 && rank >= 0 && rank < worldSize, "bad world size / rank");
    checkCudaError(cudaSetDevice(deviceId));
    comm = makeNcclCommunicatorWithId(id, idBytes, worldSize, rank);
}

// ---------------------------------------------------------------- run loop (HOT LOOP, one iteration per op)
void CudaRuntimeObj::runWithoutSyncImpl(const Graph &graph, bool validate) const {
    if (validate) graph->validateMemory();
    IT_ASSERT(graph->topo_sort(), "graph has a cycle");
    const auto &sched = graph->getSchedule();
    // resolve kernel pointers + perf records once per (graph, topology epoch) instead of two std::map
    // lookups and a workload-vector hash per op per run (reference cuda_runtime.cc:180-200)
    if (planGraphId != graph->getGraphId() || planEpoch != graph->getTopologyEpoch() || plan.size() != sched.size()) {
        plan.clear();
        plan.reserve(sched.size());
        auto &reg = KernelRegistry::getInstance();
        auto &pe = PerfEngine::getInstance();
        for (auto &st : sched) {
            const auto &op = st.ops.back();
            KernelAttrs attrs{Device::CUDA, op->getOpType().underlying()};
            for (auto &m : st.ops) reg.getKernel(KernelAttrs{Device::CUDA, m->getOpType().underlying()});  // must exist
            PlanEntry pl{reg.getKernel(attrs), pe.getPerfData({attrs, op->getOpPerfKey()})};
            plan.push_back(std::move(pl));
        }
        planGraphId = graph->getGraphId();
        planEpoch = graph->getTopologyEpoch();
    }
    // ITB_NVTX=1: one NVTX range per schedule step (nsys / ncu timelines show operator names; the reference's per-op
    // profiling table, runtime.cc:49-63, halts on CUDA -- cuda_runtime.cc:472-473)
    static const bool nvtx = [] {
        const char *e = std::getenv("ITB_NVTX");
        return e && e[0] == '1';
    }();
    b200::prepConvFilters(sched, this);
    for (size_t i = 0; i < sched.size(); ++i) {
        const auto &st = sched[i];
        struct Range {
            bool on;
            Range(bool enable, const ExecStep &s) : on(enable) {
                if (!on) return;
                string name;
                for (auto &m : s.ops) name += (name.empty() ? "" : "+") + string(m->getOpType().toString());
                nvtxRangePushA(name.c_str());
            }
            ~Range() {
                if (on) nvtxRangePop();
            }
        } range(nvtx, st);
        execStep(st, plan[i].kernel, plan[i].record ? &*plan[i].record : nullptr);
        cudaError_t err = cudaPeekAtLastError();
        if (err != cudaSuccess) {
            cudaGetLastError();
            throw Exception(string("CUDA error: ") + cudaGetErrorString(err) + " in " + st.ops.back()->toString());
        }
    }
}

// one schedule step; `kernel` / `record` = the resolved kernel of the step's last operator (nullptr: look it up)
void CudaRuntimeObj::execStep(const ExecStep &st, Kernel *kernel, const PerfRecord *record) const {
    const auto &op = st.ops.back();
    auto &reg = KernelRegistry::getInstance();
    auto single = [&](const Operator &o) {
        Kernel *k = (kernel && o == op) ? kernel : reg.getKernel(KernelAttrs{Device::CUDA, o->getOpType().underlying()});
        if (record && o == op) k->compute(o, *record, this);
        else k->compute(o, this);
    };
    switch (st.kind) {
    case ExecStep::Alias:
        // the planner made the output share the input's storage: nothing to launch
        if (op->getInputs(0)->rawPtrOrNull() == op->getOutput()->rawPtrOrNull()) break;
        [[fallthrough]];  // distinct storage (naive allocator): the ordinary copy kernel
    case ExecStep::Single:
        if (st.layout && op->getOpType() == OpType::Conv) b200::runConvBnAct(st.ops, this, st.layout);  // NHWC domain (schedule.cc)
        else if (st.layout && (op->getOpType() == OpType::MaxPool || op->getOpType() == OpType::AveragePool)) b200::runPoolNhwc(op, this);
        else single(op);  // (flat elementwise steps of the domain are layout-agnostic)
        break;
    case ExecStep::MatMulGroup: b200::runMatmulGroup(st.ops, this); break;
    case ExecStep::MatMulAdd: {
        if (!b200::matmulAddIsPlain(st.ops)) {
            // biased Linear layer and / or an activation in the chain: the wgmma epilogue, else the operators one by one
            if (!b200::runMatmulFused(st.ops, this))
                for (auto &m : st.ops) reg.getKernel(KernelAttrs{Device::CUDA, m->getOpType().underlying()})->compute(m, this);
            break;
        }
        const auto &mm = st.ops[0], &add = st.ops[1];
        auto res = add->getInputs(0) == mm->getOutput() ? add->getInputs(1) : add->getInputs(0);
        b200::runMatmul(mm, this, res, add->getOutput());
        break;
    }
    case ExecStep::SiluMul: b200::runSiluMul(st.ops[0], st.ops[1], this); break;
    case ExecStep::AttentionRope: b200::runAttentionRope(st.ops[0], st.ops[1], st.ops[2], this); break;
    case ExecStep::ConvBnAct:
        if (!b200::runConvBnAct(st.ops, this, st.layout))
            for (auto &m : st.ops) reg.getKernel(KernelAttrs{Device::CUDA, m->getOpType().underlying()})->compute(m, this);
        break;
    case ExecStep::AllReduceAddNorm:
        if (!b200::runAllReduceAddNorm(st.ops, this))
            // no NVLink peer comm (or shape outside its limits): the ordinary kernels, one by one
            for (auto &m : st.ops) reg.getKernel(KernelAttrs{Device::CUDA, m->getOpType().underlying()})->compute(m, this);
        break;
    case ExecStep::PrefillAttention: b200::runPrefillAttention(st.ops, this); break;
    }
}

void CudaRuntimeObj::run(const Graph &graph, bool tuneFlag, bool profiling) const {
    std::lock_guard<std::recursive_mutex> lock(executionMutex);
    checkCudaError(cudaSetDevice(deviceId));
    CUDAStream::Guard guard(stream);
    IT_ASSERT(!profiling, "profiling: use tune() for per-op times (reference cuda_runtime.cc:472-473 halts too)");
    if (tuneFlag) tune(graph);
    runWithoutSyncImpl(graph, true);
    checkCudaError(cudaStreamSynchronize(stream));
    checkPeerTimeout();
}

void CudaRuntimeObj::runWithoutSync(const Graph &graph) const {
    std::lock_guard<std::recursive_mutex> lock(executionMutex);
    checkCudaError(cudaSetDevice(deviceId));
    CUDAStream::Guard guard(stream);
    runWithoutSyncImpl(graph, true);
}

// per-op timing, recorded into PerfEngine (reference cuda_runtime.cc:428-464)
void CudaRuntimeObj::tune(const Graph &graph) const {
    graph->validateMemory();
    IT_ASSERT(graph->topo_sort(), "graph has a cycle");
    auto &reg = KernelRegistry::getInstance();
    auto &pe = PerfEngine::getInstance();
    for (auto &op : graph->getOperators()) {
        KernelAttrs attrs{Device::CUDA, op->getOpType().underlying()};
        PerfEngine::Key key{attrs, op->getOpPerfKey()};
        if (pe.getPerfData(key)) continue;
        PerfRecord rec = reg.getKernel(attrs)->tune(op, this);
        pe.setPerfData(key, rec);
    }
    planEpoch = ~0ull;  // re-resolve records
}

PerfRecord CudaKernelWithoutConfig::tune(const Operator &op, const RuntimeObj *context) const {
    auto rt = dynamic_cast<const CudaRuntimeObj *>(context);
    IT_ASSERT(rt != nullptr, "tune: not a CUDA runtime");
    cudaStream_t st = rt->getStream();
    cudaEvent_t a, b;
    checkCudaError(cudaEventCreate(&a));
    checkCudaError(cudaEventCreate(&b));
    const int warm = 3, rounds = 10;  // reference timeit defaults are 10/10 (include/core/common.h:92-95)
    for (int i = 0; i < warm; ++i) compute(op, context);
    checkCudaError(cudaEventRecord(a, st));
    for (int i = 0; i < rounds; ++i) compute(op, context);
    checkCudaError(cudaEventRecord(b, st));
    checkCudaError(cudaEventSynchronize(b));
    float ms = 0;
    checkCudaError(cudaEventElapsedTime(&ms, a, b));
    cudaEventDestroy(a);
    cudaEventDestroy(b);
    auto rec = make_ref<PerfRecordObj>();
    rec->time = ms / rounds;
    return rec;
}

// ---------------------------------------------------------------- CUDA-graph capture cache
vector<CudaRuntimeObj::TensorSig> CudaRuntimeObj::signature(const Graph &graph) const {
    vector<TensorSig> sig;
    sig.reserve(graph->getTensors().size());
    for (auto &t : graph->getTensors()) sig.push_back({t->rawPtrOrNull(), t->getDims(), t->getDTypeIndex()});
    return sig;
}
void CudaRuntimeObj::destroyEntry(CacheEntry &e) const {
    if (e.exec) cudaGraphExecDestroy(e.exec);
    if (e.graph) cudaGraphDestroy(e.graph);
    e.exec = nullptr;
    e.graph = nullptr;
}
void CudaRuntimeObj::clearCudaGraphCache() const {
    std::lock_guard<std::recursive_mutex> lock(executionMutex);
    for (auto &e : cache) destroyEntry(e);
    cache.clear();
}
// a failed capture leaves the stream unusable: destroy + recreate it and purge every cached graph
// (reference cuda_runtime.cc:226-250)
void CudaRuntimeObj::recoverStream() const {
    cudaGetLastError();
    for (auto &e : cache) destroyEntry(e);
    cache.clear();
    auto self = const_cast<CudaRuntimeObj *>(this);
    if (self->stream) cudaStreamDestroy(self->stream);
    self->stream = nullptr;
    checkCudaError(cudaStreamCreateWithFlags(&self->stream, cudaStreamNonBlocking));
}

void CudaRuntimeObj::runWithCudaGraph(const Graph &graph, bool syncAfter) const {
    std::lock_guard<std::recursive_mutex> lock(executionMutex);
    checkCudaError(cudaSetDevice(deviceId));
    IT_ASSERT(cacheCapacity > 0, "CUDA graph cache capacity is 0");
    graph->validateMemory();
    auto sig = signature(graph);
    for (auto it = cache.begin(); it != cache.end(); ++it) {
        if (it->graphId == graph->getGraphId() && it->topologyEpoch == graph->getTopologyEpoch() &&
            it->storageEpoch == graph->getStorageEpoch() && it->sig == sig) {
            cache.splice(cache.begin(), cache, it);  // LRU touch
            checkCudaError(cudaGraphLaunch(cache.front().exec, stream));
            if (syncAfter) {
                checkCudaError(cudaStreamSynchronize(stream));
                checkPeerTimeout();
            }
            return;
        }
    }
    // stale entries of this graph (replaced storage / changed topology) are dropped
    for (auto it = cache.begin(); it != cache.end();)
        if (it->graphId == graph->getGraphId()) {
            destroyEntry(*it);
            it = cache.erase(it);
        } else
            ++it;
    {
        // eager pass first: sizes the workspace and runs every one-time host initialisation
        // (kernel attributes, TMA driver entry point) outside the capture
        CUDAStream::Guard guard(stream);
        runWithoutSyncImpl(graph, false);
        checkCudaError(cudaStreamSynchronize(stream));
    }
    CacheEntry entry{graph->getGraphId(), graph->getTopologyEpoch(), graph->getStorageEpoch(), sig, nullptr, nullptr};
    {
        CUDAStream::Guard guard(stream);
        checkCudaError(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
        capturing = true;
        try {
            runWithoutSyncImpl(graph, false);
        } catch (...) {
            capturing = false;
            cudaGraph_t junk = nullptr;
            cudaStreamEndCapture(stream, &junk);
            if (junk) cudaGraphDestroy(junk);
            recoverStream();
            throw;
        }
        capturing = false;
        cudaError_t e = cudaStreamEndCapture(stream, &entry.graph);
        if (e != cudaSuccess || !entry.graph) {
            recoverStream();
            throw Exception(string("CUDA graph capture failed: ") + cudaGetErrorString(e));
        }
        e = cudaGraphInstantiate(&entry.exec, entry.graph, 0);
        if (e != cudaSuccess) {
            destroyEntry(entry);
            recoverStream();
            throw Exception(string("CUDA graph instantiate failed: ") + cudaGetErrorString(e));
        }
    }
    ++captureCount;
    cache.push_front(entry);
    while (cache.size() > cacheCapacity) {
        destroyEntry(cache.back());
        cache.pop_back();
    }
    checkCudaError(cudaGraphLaunch(cache.front().exec, stream));
    if (syncAfter) {
        checkCudaError(cudaStreamSynchronize(stream));
        checkPeerTimeout();
    }
}

}  // namespace infini
