// capi.cc -- the C-ABI graph / runtime handle API of include/it_b200.h (group 2).
// C spelling of the reference's pybind `backend` module (src/ffi/ffi_infinitensor.cc:441-638) and of
// GraphHandlerObj (include/core/graph_handler.h:15-159, src/core/graph_handler.cc): every handler
// method becomes itb_graph_add_op("<OpType>", inputs, outputs, attrs); exceptions become a non-zero
// return + it_b200_last_error() (pybind turns them into RuntimeError, pyinfinitensor/tests/test_api.py:21-22).
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <algorithm>

#include "b200_runtime.h"
#include "it_b200.h"
#include "operators.h"

namespace itb {
void set_error(const char *fmt, ...);
long long launches();
}  // namespace itb

using namespace infini;

// device = -1: planning-only host runtime -- graphs can be built, shape-inferred and memory-planned
// (arena bytes, copyin/copyout into host arenas) without a GPU, but nothing ever EXECUTES on it:
// run() throws.  It exists for the CPU test tier (the role of the reference's TrackingCpuRuntimeObj
// fake, test/core/test_graph.cc:14-73), not as a fallback.
class HostPlanRuntimeObj final : public RuntimeObj {
  public:
    HostPlanRuntimeObj() : RuntimeObj(Device::CPU, -1) {}
    void run(const Graph &, bool, bool) const override {
        throw Exception("planning-only host runtime: no kernels run on the host (there is no CPU fallback)");
    }
    void *alloc(size_t size) override {
        void *p = std::aligned_alloc(256, ((std::max<size_t>(size, 1) + 255) / 256) * 256);
        if (!p) throw std::bad_alloc();
        return p;
    }
    void dealloc(void *ptr) override { std::free(ptr); }
    void sync() const override {}
    void copyBlobFromCPU(void *dst, const void *src, size_t bytes) const override { std::memcpy(dst, src, bytes); }
    void copyBlobToCPU(void *dst, const void *src, size_t bytes) const override { std::memcpy(dst, src, bytes); }
    void copyBlobInsideRuntime(void *dst, const void *src, size_t bytes) const override { std::memmove(dst, src, bytes); }
    string toString() const override { return "planning-only host runtime"; }
};

struct itb_runtime {
    Ref<RuntimeObj> base;
    Ref<CudaRuntimeObj> rt;  // null for the planning-only runtime
    CudaRuntimeObj *cuda() const {
        IT_ASSERT(rt != nullptr, "planning-only host runtime: this call needs a CUDA runtime (no CPU fallback)");
        return rt.get();
    }
};
struct itb_graph {
    itb_runtime *owner;
    Ref<RuntimeObj> base;
    Ref<CudaRuntimeObj> rt;
    CudaRuntimeObj *cuda() const {
        IT_ASSERT(rt != nullptr, "planning-only host runtime: this call needs a CUDA runtime (no CPU fallback)");
        return rt.get();
    }
    Graph g;
    std::unordered_map<TensorObj *, itb_tensor> ids;
    itb_tensor idOf(const Tensor &t) {
        auto it = ids.find(t.get());
        if (it != ids.end()) return it->second;
        // tensors created by operator constructors are appended to the graph: index them lazily
        const auto &ts = g->getTensors();
        for (size_t i = 0; i < ts.size(); ++i) ids.emplace(ts[i].get(), (itb_tensor)i);
        return ids.at(t.get());
    }
    Tensor get(itb_tensor id) {
        if (id < 0) return nullptr;
        IT_ASSERT((size_t)id < g->getTensors().size(), "bad tensor id");
        return g->getTensors()[(size_t)id];
    }
};

#define ITB_TRY(...)                                                                           \
    try {                                                                                      \
        __VA_ARGS__;                                                                           \
        return 0;                                                                              \
    } catch (const std::bad_alloc &) {                                                         \
        itb::set_error("out of device memory");                                                \
        return 2;                                                                              \
    } catch (const std::exception &e) {                                                        \
        itb::set_error("%s", e.what());                                                        \
        return 1;                                                                              \
    }

extern "C" {

int itb_runtime_create(int device, int64_t cap, itb_runtime **out) {
    ITB_TRY({
        auto r = new itb_runtime;
        if (device < 0) {
            r->base = make_ref<HostPlanRuntimeObj>();
        } else {
            r->rt = make_ref<CudaRuntimeObj>(device, (size_t)cap);
            r->base = r->rt;
        }
        *out = r;
    })
}
int itb_runtime_destroy(itb_runtime *rt) { ITB_TRY(delete rt) }
int itb_runtime_init_comm(itb_runtime *rt, const char *name, int world, int rank) {
    ITB_TRY(rt->cuda()->initComm(name, world, rank))
}
int itb_runtime_init_comm_with_id(itb_runtime *rt, const void *id, int n, int world, int rank) {
    ITB_TRY(rt->cuda()->initCommWithId(id, n, world, rank))
}
int itb_runtime_nccl_unique_id(void *out, int n) {
    try {
        return ncclUniqueIdBytes(out, n);
    } catch (const std::exception &e) {
        itb::set_error("%s", e.what());
        return 0;
    }
}
int itb_runtime_p2p_export(itb_runtime *rt, void *handle64) { ITB_TRY(rt->cuda()->p2pExport(handle64)) }
int itb_runtime_p2p_import(itb_runtime *rt, const void *all, int world, int rank) {
    ITB_TRY(rt->cuda()->p2pImport(all, world, rank))
}
int64_t itb_runtime_cuda_graph_cache_size(itb_runtime *rt) { return rt->rt ? (int64_t)rt->rt->getCudaGraphCacheSize() : 0; }
int64_t itb_runtime_cuda_graph_capture_count(itb_runtime *rt) { return rt->rt ? (int64_t)rt->rt->getCudaGraphCaptureCount() : 0; }
int itb_runtime_clear_cuda_graph_cache(itb_runtime *rt) { ITB_TRY(rt->cuda()->clearCudaGraphCache()) }
int64_t itb_runtime_kernel_launches(itb_runtime *) { return itb::launches(); }
void *itb_runtime_stream(itb_runtime *rt) { return rt->rt ? (void *)rt->rt->getStream() : nullptr; }

int itb_graph_create(itb_runtime *rt, itb_graph **out) {
    ITB_TRY({
        auto g = new itb_graph;
        g->owner = rt;
        g->rt = rt->rt;
        g->base = rt->base;
        g->g = make_ref<GraphObj>(rt->base);
        *out = g;
    })
}
int itb_graph_destroy(itb_graph *g) { ITB_TRY(delete g) }

int itb_graph_tensor(itb_graph *g, const int *dims, int rank, int dtype, itb_tensor *out) {
    ITB_TRY({
        IT_ASSERT(DataType(dtype).getSize() > 0, "unsupported dtype " + std::to_string(dtype));
        auto t = g->g->addTensor(Shape(dims, dims + rank), DataType(dtype));
        *out = g->idOf(t);
    })
}
int itb_tensor_set_weight(itb_graph *g, itb_tensor t) { ITB_TRY(g->get(t)->setWeight()) }
int itb_tensor_set_input(itb_graph *g, itb_tensor t) { ITB_TRY(g->get(t)->setInput()) }
int itb_tensor_set_output(itb_graph *g, itb_tensor t) { ITB_TRY(g->get(t)->setOutput()) }
int itb_tensor_rank(itb_graph *g, itb_tensor t) {
    try {
        return (int)g->get(t)->getRank();
    } catch (const std::exception &e) {
        itb::set_error("%s", e.what());
        return -1;
    }
}
int itb_tensor_shape(itb_graph *g, itb_tensor t, int *dims_out) {
    ITB_TRY({
        auto &d = g->get(t)->getDims();
        for (size_t i = 0; i < d.size(); ++i) dims_out[i] = d[i];
    })
}
int itb_tensor_dtype(itb_graph *g, itb_tensor t) {
    try {
        return g->get(t)->getDTypeIndex();
    } catch (const std::exception &e) {
        itb::set_error("%s", e.what());
        return -1;
    }
}
int64_t itb_tensor_bytes(itb_graph *g, itb_tensor t) {
    try {
        return (int64_t)g->get(t)->getBytes();
    } catch (const std::exception &e) {
        itb::set_error("%s", e.what());
        return -1;
    }
}
void *itb_tensor_device_ptr(itb_graph *g, itb_tensor t) {
    try {
        return g->get(t)->rawPtrOrNull();
    } catch (...) {
        return nullptr;
    }
}
int itb_tensor_copyin(itb_graph *g, itb_tensor t, const void *host, int64_t bytes) {
    ITB_TRY(g->get(t)->copyin(host, (size_t)bytes))
}
int itb_tensor_copyout(itb_graph *g, itb_tensor t, void *host, int64_t bytes) {
    ITB_TRY(g->get(t)->copyout(host, (size_t)bytes))
}
int itb_tensor_copyin_async(itb_graph *g, itb_tensor t, const void *host, int64_t bytes) {
    ITB_TRY({
        auto T = g->get(t);
        IT_ASSERT((size_t)bytes == T->getBytes(), "copyin: size mismatch");
        g->cuda()->copyBlobFromCPUAsync(T->getRawDataPtr<void *>(), host, (size_t)bytes);
    })
}
int itb_tensor_copyout_async(itb_graph *g, itb_tensor t, void *host, int64_t bytes) {
    ITB_TRY({
        auto T = g->get(t);
        IT_ASSERT((size_t)bytes == T->getBytes(), "copyout: size mismatch");
        g->cuda()->copyBlobToCPUAsync(host, T->getRawDataPtr<void *>(), (size_t)bytes);
    })
}

static vector<int> ivec(const int64_t *a, int from, int n) {
    vector<int> v;
    for (int i = 0; i < n; ++i) v.push_back((int)a[from + i]);
    return v;
}

static Operator build_op(itb_graph *h, const string &name, const TensorVec &in, TensorVec &out, const int64_t *ia,
                         int ni, const double *fa, int nf) {
    GraphObj *gp = nullptr;  // ops are built detached, then connected (so given outputs are honoured)
    Graph g = h->g;
    auto o0 = out.empty() ? nullptr : out[0];
    auto need = [&](size_t n) { IT_ASSERT(in.size() >= n, name + ": expected at least " + std::to_string(n) + " inputs"); };
    auto I = [&](int i, int64_t def = 0) { return i < ni ? ia[i] : def; };
    auto F = [&](int i, double def = 0) { return i < nf ? fa[i] : def; };
    (void)gp;
    OpType t = OpType::fromString(name);
    switch (t.underlying()) {
    case OpType::MatMul:
        need(2);
    {
        const bool scaled = I(3, 0) != 0;  // extension: the last input is the FP8 weight's per-column scale
        need(scaled ? 3 : 2);
        const size_t nb = in.size() - (scaled ? 1 : 0);
        return g->addOp<MatmulObj>(in[0], in[1], o0, (bool)I(0), (bool)I(1), nb > 2 ? in[2] : nullptr, (ActType)I(2), "default",
                                   scaled ? in.back() : nullptr);
    }
    case OpType::MatMulNBits:
    {
        // inputs A, B, scales, then the optional zero_points, g_idx, bias that are present; iattrs K, N, bits, block_size and
        // one presence flag per optional input
        need(3);
        size_t next = 3;
        auto opt = [&](int flag) -> Tensor {
            if (!I(flag)) return nullptr;
            need(next + 1);
            return in[next++];
        };
        Tensor zp = opt(4), gidx = opt(5), bias = opt(6);
        IT_ASSERT(next == in.size(), "MatMulNBits: " + std::to_string(in.size()) + " inputs do not match the presence flags");
        return g->addOp<MatMulNBitsObj>(in[0], in[1], in[2], zp, o0, (int)I(0), (int)I(1), (int)I(2, 4), (int)I(3), gidx, bias);
    }
    case OpType::Conv:
        need(2);
        return g->addOp<ConvObj>(in[0], in[1], o0, (int)I(0), (int)I(1), (int)I(2, 1), (int)I(3, 1), (int)I(4, 1),
                                 (int)I(5, 1));
    case OpType::AttentionKVCache:  // iattr 0: per-row positions, 1: sliding window, 2: rolling cache (all extensions)
        need(6);
        IT_ASSERT(in.size() == 6 || in.size() == 8, "AttentionKVCache: 6 inputs, or 8 with an FP8 cache's k_scale / v_scale");
        return g->addOp<AttentionKVCacheObj>(in[0], in[1], in[2], in[3], in[4], in[5], o0, (bool)I(0, 0),
                                             in.size() == 8 ? in[6] : nullptr, in.size() == 8 ? in[7] : nullptr, (int)I(1, 0),
                                             (bool)I(2, 0));
    case OpType::Softmax: need(1); return g->addOp<SoftmaxObj>(in[0], o0, (int)I(0, -1));
    case OpType::LayerNormalization:
        need(2);
        return g->addOp<LayerNormObj>(in[0], in[1], o0, in.size() > 2 ? in[2] : nullptr, (float)F(0, 1e-5),
                                      (int)I(0, -1), (int)I(1, 1));
    case OpType::RMSNorm: need(2); return g->addOp<RMSNormObj>(in[0], in[1], o0);
    case OpType::RoPE:  // iattr 0: dim_head (extension); an optional third input: the inv_freq table (extension)
        need(2);
        IT_ASSERT(in.size() <= 3, "RoPE: at most 3 inputs (pos, input, inv_freq)");
        return g->addOp<RoPEObj>(in[0], in[1], o0, (int)I(0, 128), in.size() > 2 ? in[2] : nullptr);
    case OpType::LeakyRelu: need(1); return g->addOp<LeakyReluObj>(in[0], o0, (float)F(0, 0.01));
    case OpType::Elu: need(1); return g->addOp<EluObj>(in[0], o0, (float)F(0, 1.0));
    case OpType::Relu: case OpType::Sigmoid: case OpType::Tanh: case OpType::Gelu: case OpType::Silu:
    case OpType::Erf: case OpType::Neg: case OpType::Abs: case OpType::Sqrt: case OpType::HardSigmoid:
    case OpType::HardSwish: case OpType::Exp: case OpType::Identity:
        need(1);
    {
        auto op = make_ref<UnaryObj>(t, g.get(), in[0], o0);
        g->addOperator(op);
        return op;
    }
    case OpType::Add: case OpType::Sub: case OpType::Mul: case OpType::Div: case OpType::Pow: case OpType::Min:
    case OpType::Max: case OpType::Less: case OpType::Equal: case OpType::Greater:
        need(2);
    {
        auto op = make_ref<ElementWiseObj>(t, g.get(), in[0], in[1], o0);
        g->addOperator(op);
        return op;
    }
    case OpType::Transpose: need(1); return g->addOp<TransposeObj>(in[0], o0, ivec(ia, 0, ni));
    case OpType::DepthToSpace: need(1); return g->addOp<DepthToSpaceObj>(in[0], o0, (int)I(0, 1), I(1, 0) ? "CRD" : "DCR");
    case OpType::Concat: need(1); return g->addOp<ConcatObj>(in, o0, (int)I(0));
    case OpType::Split: {
        need(1);
        std::optional<TensorVec> outs;
        bool given = false;
        for (auto &o : out) given = given || o;
        if (given) outs = out;
        if (I(1) > 0) return g->addOp<SplitObj>(in[0], outs, (int)I(0), (int)I(1));
        return g->addOp<SplitObj>(in[0], outs, (int)I(0), ivec(ia, 2, ni - 2));
    }
    case OpType::Gather: need(2); return g->addOp<GatherObj>(in[0], in[1], o0, (int)I(0));
    case OpType::Reshape: need(1); return g->addOp<ReshapeObj>(in[0], o0, ivec(ia, 0, ni));
    case OpType::Flatten: need(1); return g->addOp<FlattenObj>(in[0], o0, (int)I(0, 1));
    case OpType::Squeeze: need(1); return g->addOp<SqueezeObj>(in[0], o0, ivec(ia, 0, ni));
    case OpType::Unsqueeze: need(1); return g->addOp<UnsqueezeObj>(in[0], o0, ivec(ia, 0, ni));
    case OpType::Cast: need(1); return g->addOp<CastObj>(in[0], o0, DataType((int)I(0, 1)));
    case OpType::Where: need(3); return g->addOp<WhereObj>(in[0], in[1], in[2], o0);
    case OpType::Expand: need(1); return g->addOp<ExpandObj>(in[0], o0, ivec(ia, 0, ni));
    case OpType::ReduceMean: case OpType::ReduceSum: {
        need(1);
        std::optional<vector<int>> axes;
        if (ni > 1) axes = ivec(ia, 1, ni - 1);
        if (t == OpType::ReduceMean) return g->addOp<ReduceMeanObj>(in[0], o0, axes, (bool)I(0, 1));
        return g->addOp<ReduceSumObj>(in[0], o0, axes, (bool)I(0, 1));
    }
    case OpType::Slice: {
        // iattrs: n, starts[n], ends[n], has_axes, axes[n]?, has_steps, steps[n]?
        need(1);
        int n = (int)I(0), p = 1;
        auto starts = ivec(ia, p, n);
        p += n;
        auto ends = ivec(ia, p, n);
        p += n;
        std::optional<vector<int>> axes, steps;
        if (I(p++)) {
            axes = ivec(ia, p, n);
            p += n;
        }
        if (I(p++)) steps = ivec(ia, p, n);
        return g->addOp<SliceObj>(in[0], o0, starts, ends, axes, steps);
    }
    case OpType::Pad: {
        // iattrs: npads, pads[npads], has_axes, axes[npads/2]?
        need(1);
        int n = (int)I(0);
        auto pads = ivec(ia, 1, n);
        std::optional<vector<int>> axes;
        if (I(1 + n)) axes = ivec(ia, 2 + n, n / 2);
        return g->addOp<PadObj>(in[0], o0, pads, axes);
    }
    case OpType::MaxPool: case OpType::AveragePool: {
        need(1);
        IT_ASSERT(ni >= 8, "pooling needs kh,kw,dh,dw,ph,pw,sh,sw[,ceilMode]");
        if (t == OpType::MaxPool)
            return g->addOp<MaxPoolObj>(in[0], o0, (int)I(0), (int)I(1), (int)I(2), (int)I(3), (int)I(4), (int)I(5),
                                        (int)I(6), (int)I(7), (int)I(8));
        return g->addOp<AvgPoolObj>(in[0], o0, (int)I(0), (int)I(1), (int)I(2), (int)I(3), (int)I(4), (int)I(5),
                                    (int)I(6), (int)I(7), (int)I(8));
    }
    case OpType::BatchNormalization:
        need(5);
        return g->addOp<BatchNormObj>(in[0], o0, in[1], in[2], in[3], in[4], (float)F(0, 0.9), (float)F(1, 1e-5),
                                      (bool)I(0));
    case OpType::AllReduceSum: case OpType::AllReduceProd: case OpType::AllReduceMin: case OpType::AllReduceMax:
    case OpType::AllReduceAvg:
        need(1);
        return g->addOp<AllReduceBaseObj>(t, in[0], o0);
    case OpType::AllGather: {
        need(1);
        std::optional<TensorVec> outs;
        bool given = false;
        for (auto &o : out) given = given || o;
        if (given) outs = out;
        return g->addOp<AllGatherObj>(in[0], outs, (int)I(0));
    }
    default: IT_ASSERT(false, "unsupported operator type '" + name + "'");
    }
    return nullptr;
}

int itb_graph_add_op(itb_graph *g, const char *op_type, const itb_tensor *inputs, int n_inputs, itb_tensor *outputs,
                     int n_outputs, const int64_t *iattrs, int n_iattrs, const double *fattrs, int n_fattrs) {
    ITB_TRY({
        TensorVec in, out;
        for (int i = 0; i < n_inputs; ++i)
            if (inputs[i] >= 0) in.push_back(g->get(inputs[i]));
        for (int i = 0; i < n_outputs; ++i) out.push_back(g->get(outputs[i]));
        auto op = build_op(g, op_type, in, out, iattrs, n_iattrs, fattrs, n_fattrs);
        IT_ASSERT((int)op->getOutputs().size() <= n_outputs || n_outputs == 0,
                  string(op_type) + ": output array too small");
        for (int i = 0; i < n_outputs && i < (int)op->getOutputs().size(); ++i) outputs[i] = g->idOf(op->getOutput(i));
    })
}

int itb_graph_num_ops(itb_graph *g) { return (int)g->g->getOperators().size(); }
int itb_graph_op_type(itb_graph *g, int index, char *buf, int buf_len) {
    ITB_TRY({
        IT_ASSERT(index >= 0 && index < (int)g->g->getOperators().size(), "bad op index");
        snprintf(buf, buf_len, "%s", g->g->getOperators()[index]->getOpType().toString());
    })
}
int itb_graph_num_steps(itb_graph *g) {
    try {
        return (int)g->g->getSchedule().size();
    } catch (const std::exception &e) {
        itb::set_error("%s", e.what());
        return -1;
    }
}
int itb_graph_step(itb_graph *g, int index, char *buf, int buf_len) {
    ITB_TRY({
        const auto &sc = g->g->getSchedule();
        IT_ASSERT(index >= 0 && index < (int)sc.size(), "bad step index");
        static const char *kinds[] = {"Single", "Alias", "MatMulGroup", "MatMulAdd", "SiluMul", "AttentionRope", "AllReduceAddNorm", "ConvBnAct", "PrefillAttention"};
        std::string s = kinds[(int)sc[index].kind];
        s += ":";
        for (size_t i = 0; i < sc[index].ops.size(); ++i) s += (i ? "+" : "") + std::string(sc[index].ops[i]->getOpType().toString());
        // NHWC domain: "@nhwc" = operands and result channel-innermost, "@>nhwc" = enters the domain, "@nhwc>" = leaves it
        static const char *lay[] = {"", "@nhwc>", "@>nhwc", "@nhwc"};
        s += lay[sc[index].layout & 3];
        snprintf(buf, buf_len, "%s", s.c_str());
    })
}
int itb_graph_topo_sort(itb_graph *g) { ITB_TRY(IT_ASSERT(g->g->topo_sort(), "graph has a cycle")) }
int itb_graph_shape_infer(itb_graph *g) { ITB_TRY(g->g->shape_infer()) }
int itb_graph_optimize(itb_graph *g) { ITB_TRY(g->g->optimize()) }
int itb_graph_data_malloc(itb_graph *g, int naive, int64_t pool) { ITB_TRY(g->g->dataMalloc(naive != 0, (size_t)pool)) }
int itb_graph_run(itb_graph *g) { ITB_TRY(g->base->run(g->g)) }
int itb_graph_run_without_sync(itb_graph *g) { ITB_TRY(g->cuda()->runWithoutSync(g->g)) }
int itb_graph_run_with_cudagraph(itb_graph *g) { ITB_TRY(g->cuda()->runWithCudaGraph(g->g, true)) }
int itb_graph_launch_cudagraph_async(itb_graph *g) { ITB_TRY(g->cuda()->runWithCudaGraph(g->g, false)) }
int itb_graph_tune(itb_graph *g) { ITB_TRY(g->base->run(g->g, true)) }
int itb_graph_sync(itb_graph *g) { ITB_TRY(g->base->sync()) }
double itb_graph_get_perf_time(itb_graph *g) {
    try {
        return g->base->getPerfTime(g->g);
    } catch (...) {
        return -1.0;
    }
}
int itb_perf_engine_save(const char *path) { ITB_TRY(PerfEngine::getInstance().savePerfEngineData(path)) }
int itb_perf_engine_load(const char *path) { ITB_TRY(PerfEngine::getInstance().loadPerfEngineData(path)) }
int64_t itb_perf_engine_size(void) { return (int64_t)PerfEngine::getInstance().size(); }
void itb_perf_engine_clear(void) { PerfEngine::getInstance().clear(); }

int64_t itb_graph_arena_bytes(itb_graph *g, int which) {
    return (int64_t)(which == 0 ? g->g->getWeightArenaBytes() : g->g->getActivationArenaBytes());
}

}  // extern "C"
