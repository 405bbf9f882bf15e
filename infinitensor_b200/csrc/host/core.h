// core.h -- host contract of the B200 backend: the executor-side types the kernels plug into.
//
// Written from scratch to the SEMANTICS of the reference's core (names and meaning kept so that
// reference tests / frontends read the same; citations relative to /root/reference):
//   Exception / IT_ASSERT ........ include/core/common.h:44-55
//   DataType (ONNX indices) ...... include/core/data_type.h:6-23
//   TensorObj .................... include/core/tensor.h, tensor_base.h:38-43
//   OperatorObj / OpType ......... include/core/operator.h:46-129, include/core/op_type.h
//   GraphObj (topo sort, planner)  include/core/graph.h:38-206, src/core/graph.cc:152-182,341-576
//   LazyAllocator ................ src/core/lazy_allocator.cc (best-fit arena, 256 B alignment :13)
//   Kernel / KernelRegistry / REGISTER_KERNEL / PerfEngine ... include/core/kernel.h:32-205,
//                                  include/core/perf_engine.h:8-48
//   RuntimeObj ................... include/core/runtime.h:38-101
#pragma once
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <sstream>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <variant>
#include <vector>

namespace infini {

using std::string;
using std::vector;
template <typename T> using Ref = std::shared_ptr<T>;
template <typename T> using WRef = std::weak_ptr<T>;
template <typename T, typename... A> Ref<T> make_ref(A &&...a) { return std::make_shared<T>(std::forward<A>(a)...); }
template <typename T, typename U> Ref<T> as(const Ref<U> &r) { return std::dynamic_pointer_cast<T>(r); }

class Exception : public std::runtime_error {
  public:
    explicit Exception(const string &msg) : std::runtime_error(msg) {}
};

#define IT_ASSERT(cond, ...)                                                                   \
    do {                                                                                       \
        if (!(cond)) {                                                                         \
            std::ostringstream os__;                                                           \
            os__ << "Assertion failed: " #cond " at " << __FILE__ << ":" << __LINE__ << " " << string(__VA_ARGS__); \
            throw ::infini::Exception(os__.str());                                             \
        }                                                                                      \
    } while (0)
#define IT_TODO_HALT() IT_ASSERT(false, "Unimplemented")
#define IT_TODO_HALT_MSG(msg) IT_ASSERT(false, msg)

using Shape = vector<int>;
using UidBaseType = int;

// ---------------------------------------------------------------- DataType
class DataType {
    int index;

  public:
    static const DataType Undefine, Float32, UInt8, Int8, UInt16, Int16, Int32, Int64, String, Bool, Float16,
        Double, UInt32, UInt64, BFloat16, Float8E4M3FN;  // 17 = ONNX FLOAT8E4M3FN: quantised weights (SURVEY 8(f-4); not in the reference)
    constexpr DataType(int index = 1) : index(index) {}
    bool operator==(const DataType &o) const { return index == o.index; }
    bool operator!=(const DataType &o) const { return index != o.index; }
    bool operator<(const DataType &o) const { return index < o.index; }
    int getIndex() const { return index; }
    size_t getSize() const {
        static const size_t sz[] = {0, 4, 1, 1, 2, 2, 4, 8, 0, 1, 2, 8, 4, 8, 0, 0, 2, 1};
        return index >= 0 && index <= 17 ? sz[index] : 0;
    }
    string toString() const {
        static const char *nm[] = {"Undefine", "Float32", "UInt8", "Int8", "UInt16", "Int16", "Int32", "Int64",
                                   "String", "Bool", "Float16", "Double", "UInt32", "UInt64", "?", "?", "BFloat16", "Float8E4M3FN"};
        return index >= 0 && index <= 17 ? nm[index] : "?";
    }
    bool isFloat() const { return index == 1 || index == 10 || index == 16; }
};

enum class Device { CPU = 1, CUDA, BANG, INTELCPU, KUNLUN, ASCEND };
enum class ActType { None, Relu, Sigmoid, Tanh };

// ---------------------------------------------------------------- OpType
struct OpType {
    using underlying_t = uint16_t;
    enum : underlying_t {
        Unknown, Abs, Add, AllGather, AllReduceAvg, AllReduceMax, AllReduceMin, AllReduceProd, AllReduceSum,
        AttentionKVCache, AveragePool, BatchNormalization, Cast, Concat, Conv, DepthToSpace, Div, Elu, Equal, Erf, Exp,
        Expand, Flatten, Gather, Gelu, Greater, HardSigmoid, HardSwish, Identity, LayerNormalization, LeakyRelu, Less, MatMul,
        Max, MaxPool, Min, Mul, Neg, Pad, Pow, RMSNorm, ReduceMean, ReduceSum, Relu, Reshape, RoPE, Sigmoid, Silu,
        Slice, Softmax, Split, Sqrt, Squeeze, Sub, Tanh, Transpose, Unsqueeze, Where,
        MatMulNBits,  // (extensions after the reference's alphabetical list, so that its numbering stays)
        NumOpTypes
    } type;
    constexpr OpType(decltype(type) t = Unknown) : type(t) {}
    constexpr explicit OpType(underlying_t v) : type((decltype(type))v) {}
    constexpr underlying_t underlying() const { return type; }
    bool operator==(OpType o) const { return type == o.type; }
    bool operator!=(OpType o) const { return type != o.type; }
    bool operator<(OpType o) const { return type < o.type; }
    const char *toString() const;
    static OpType fromString(const string &s);  // Unknown if not found
};

// ---------------------------------------------------------------- forward decls
class RuntimeObj;
class TensorObj;
class OperatorObj;
class GraphObj;
using Runtime = Ref<RuntimeObj>;
using Tensor = Ref<TensorObj>;
using Operator = Ref<OperatorObj>;
using Graph = Ref<GraphObj>;
using TensorVec = vector<Tensor>;
using OpVec = vector<Operator>;

// ---------------------------------------------------------------- Blob: device memory owner / view
class BlobObj {
    Runtime runtime;
    void *ptr;
    size_t bytes;
    Ref<BlobObj> owner;  // views keep the arena root alive (reference src/core/blob.cc:12-42)
  public:
    BlobObj(Runtime rt, void *ptr, size_t bytes, Ref<BlobObj> owner = nullptr)
        : runtime(std::move(rt)), ptr(ptr), bytes(bytes), owner(std::move(owner)) {}
    ~BlobObj();
    BlobObj(const BlobObj &) = delete;
    BlobObj &operator=(const BlobObj &) = delete;
    template <typename T> T getPtr() const { return reinterpret_cast<T>(ptr); }
    size_t getBytes() const { return bytes; }
};
using Blob = Ref<BlobObj>;

// ---------------------------------------------------------------- Tensor
class TensorObj : public std::enable_shared_from_this<TensorObj> {
    friend class GraphObj;
    Shape shape;
    DataType dtype;
    Runtime runtime;
    Blob data;
    UidBaseType guid, fuid;
    bool weightFlag = false, inputFlag = false, outputFlag = false;
    WRef<OperatorObj> source;
    vector<WRef<OperatorObj>> targets;

  public:
    TensorObj(Shape shape, DataType dtype, Runtime runtime);
    const Shape &getDims() const { return shape; }
    void setShape(Shape s) { shape = std::move(s); }
    size_t getRank() const { return shape.size(); }
    Shape getStride() const;
    size_t size() const;
    size_t getBytes() const { return size() * dtype.getSize(); }
    DataType getDType() const { return dtype; }
    int getDTypeIndex() const { return dtype.getIndex(); }
    Runtime getRuntime() const { return runtime; }
    UidBaseType getGuid() const { return guid; }
    UidBaseType getFuid() const { return fuid; }
    // fusion and alias decisions read these flags (isOutput / isWeight / isInput), so changing one must invalidate every cached
    // schedule, dispatch plan and captured CUDA graph: a process-wide counter the graphs fold into their topology epoch
    static uint64_t &flagsEpoch() {
        static uint64_t e = 0;
        return e;
    }
    void setWeight() { if (!weightFlag) ++flagsEpoch(); weightFlag = true; }
    void setInput() { if (!inputFlag) ++flagsEpoch(); inputFlag = true; }
    void setOutput() { if (!outputFlag) ++flagsEpoch(); outputFlag = true; }
    bool isWeight() const { return weightFlag; }
    bool isInput() const { return inputFlag; }
    bool isOutput() const { return outputFlag; }
    bool hasData() const { return data != nullptr; }
    void setDataBlob(const Blob &b) { data = b; }
    Blob getDataBlob() const { return data; }
    void freeData() { data = nullptr; }
    template <typename T> T getRawDataPtr() const {
        IT_ASSERT(data != nullptr, "tensor has no storage (call data_malloc first)");
        return data->getPtr<T>();
    }
    void *rawPtrOrNull() const { return data ? data->getPtr<void *>() : nullptr; }
    void dataMalloc();  // standalone allocation (outside a graph plan)
    void copyin(const void *host, size_t bytes);
    void copyout(void *host, size_t bytes) const;
    Operator getSource() const { return source.lock(); }
    OpVec getTargets() const;
    bool hasTarget() const { return !targets.empty(); }
    string toString() const;
};

// ---------------------------------------------------------------- Operator
using HashType = uint64_t;
struct KernelAttrs {
    Device device;
    OpType::underlying_t op;
    bool operator<(const KernelAttrs &o) const { return std::tie(device, op) < std::tie(o.device, o.op); }
};
struct OpPerfKey {
    HashType hash;
    OpType::underlying_t opType;
    vector<int> attrs;
    bool operator<(const OpPerfKey &o) const {
        return std::tie(hash, opType, attrs) < std::tie(o.hash, o.opType, o.attrs);
    }
};

class OperatorObj : public std::enable_shared_from_this<OperatorObj> {
    friend class GraphObj;

  protected:
    OpType type;
    TensorVec inputs, outputs;
    vector<WRef<OperatorObj>> predecessors, successors;
    UidBaseType guid;

  public:
    OperatorObj(OpType type, TensorVec inputs, TensorVec outputs);
    virtual ~OperatorObj() = default;
    virtual std::optional<vector<Shape>> inferShape(const TensorVec &inputs) = 0;
    virtual vector<DataType> inferDataType(const TensorVec &inputs) const;
    virtual string toString() const;
    virtual int numInputs() const { return (int)inputs.size(); }
    virtual int numOutputs() const { return (int)outputs.size(); }
    virtual vector<int> getWorkloadVector() const;
    virtual vector<int> getOpAttrVector() const { return {(int)type.underlying()}; }
    std::optional<vector<Shape>> inferShape() { return inferShape(inputs); }
    bool checkValid(GraphObj *graph);
    OpPerfKey getOpPerfKey() const;
    OpType getOpType() const { return type; }
    const TensorVec &getInputs() const { return inputs; }
    const TensorVec &getOutputs() const { return outputs; }
    Tensor getInputs(size_t i) const { return inputs.at(i); }
    Tensor getOutput() const {
        IT_ASSERT(outputs.size() == 1, "Unimplemented");
        return outputs[0];
    }
    Tensor getOutput(size_t i) const { return outputs.at(i); }
    DataType getDType() const { return getInputs(0)->getDType(); }
    DataType getOutDType() const { return outputs[0]->getDType(); }
    UidBaseType getGuid() const { return guid; }
    OpVec getPredecessors() const;
    OpVec getSuccessors() const;
};

// ---------------------------------------------------------------- Kernel plugin API
struct PerfRecordObj {
    double time = 0;  // ms
    virtual ~PerfRecordObj() = default;
    virtual int type() const { return 0; }  // JSON "type" (perf_engine.cc:7-62)
};
using PerfRecord = Ref<PerfRecordObj>;
// what MatMul's tune() measured best for one (shape, dtype) key -- the counterpart of the reference's MatmulCublasPerfRecordObj
// (matmul.cc:12-24: the cuBLAS algorithm index): which of this repo's GEMM kernels, and the skinny kernel's tile width
struct MatmulPerfRecordObj : PerfRecordObj {
    int impl = 0;  // 0 = the production dispatch order, 1 = gemm_skinny (mma.sync, cluster split-K), 2 = gemm_tc (wgmma), 3 = gemm_simt
    int nb = 0;    // skinny: 64-column boxes per tile (1 / 2; 0 = automatic)
    int type() const override { return 1; }
};

class Kernel {
  public:
    virtual ~Kernel() = default;
    virtual void compute(const Operator &op, const PerfRecord &record, const RuntimeObj *context) const = 0;
    virtual void compute(const Operator &op, const RuntimeObj *context) const = 0;
    virtual PerfRecord tune(const Operator &op, const RuntimeObj *context) const = 0;
};

class KernelRegistry {
    std::map<KernelAttrs, std::pair<Kernel *const, const string>> kernels;
    int nKernels = 0;

  public:
    ~KernelRegistry();
    static KernelRegistry &getInstance();
    bool registerKernel(const KernelAttrs &key, Kernel *kernel, string name);  // duplicate key -> throws
    Kernel *getKernel(const KernelAttrs &attrs) const;                          // missing -> throws
    bool hasKernel(const KernelAttrs &attrs) const { return kernels.count(attrs) > 0; }
    const string &getKernelName(const KernelAttrs &attrs) const;
    int numKernels() const { return nKernels; }
};

#define _REGISTER_KERNEL_1(device, opType, kernel, name, cnt)                                  \
    namespace infini {                                                                         \
    static const bool _register_kernel_##cnt = KernelRegistry::getInstance().registerKernel(   \
        KernelAttrs{device, OpType(opType).underlying()}, new kernel(), name);                 \
    }
#define _REGISTER_KERNEL_0(device, opType, kernel, name, cnt) _REGISTER_KERNEL_1(device, opType, kernel, name, cnt)
#define REGISTER_KERNEL(device, opType, kernel, name) _REGISTER_KERNEL_0(device, opType, kernel, name, __COUNTER__)

class PerfEngine {
  public:
    using Key = std::pair<KernelAttrs, OpPerfKey>;
    static PerfEngine &getInstance();
    std::optional<PerfRecord> getPerfData(const Key &key) const;
    void setPerfData(const Key &key, PerfRecord record);  // duplicate -> throws (perf_engine.h:40-43)
    size_t size() const { return data.size(); }
    void clear() { data.clear(); }
    // JSON in the layout nlohmann gives the reference's map (src/core/perf_engine.cc:7-62): files are interchangeable.
    //   {"data": [ [ [[device, opType], {"attrs": [...], "hashType": h, "opType": o}], {"data": ms, "type": 0} ], ... ]}
    // load REPLACES the table, like the reference's set_data; the time is read as a double (the reference reads it back
    // as an int, quirk q13 -- not reproduced).
    void savePerfEngineData(const string &path) const;
    void loadPerfEngineData(const string &path);

  private:
    std::map<Key, PerfRecord> data;
};

// ---------------------------------------------------------------- Runtime
class RuntimeObj : public std::enable_shared_from_this<RuntimeObj> {
  protected:
    Device device;
    int deviceId;

  public:
    RuntimeObj(Device device, int deviceId = 0) : device(device), deviceId(deviceId) {}
    virtual ~RuntimeObj() = default;
    RuntimeObj(const RuntimeObj &) = delete;
    virtual void run(const Graph &graph, bool tune = false, bool profiling = false) const = 0;
    virtual void *alloc(size_t size) = 0;
    virtual void dealloc(void *ptr) = 0;
    virtual void sync() const = 0;
    virtual void copyBlobFromCPU(void *dst, const void *src, size_t bytes) const = 0;
    virtual void copyBlobToCPU(void *dst, const void *src, size_t bytes) const = 0;
    virtual void copyBlobInsideRuntime(void *dst, const void *src, size_t bytes) const = 0;
    virtual double getPerfTime(const Graph &graph) const;
    virtual string toString() const = 0;
    Device getDevice() const { return device; }
    int getDeviceId() const { return deviceId; }
    bool isCuda() const { return device == Device::CUDA; }
    virtual size_t getAlignment() const { return 256; }
};

// ---------------------------------------------------------------- LazyAllocator (offline arena planner)
class LazyAllocator {
    size_t alignment;
    size_t used = 0, peak = 0;
    std::map<size_t, size_t> freeByAddr;           // offset -> size
    std::set<std::pair<size_t, size_t>> freeBySize;  // (size, offset)
    void insertFree(size_t off, size_t size);
    void eraseFree(size_t off, size_t size);

  public:
    explicit LazyAllocator(size_t alignment = 256) : alignment(alignment) {}
    size_t getAlignedSize(size_t size) const { return ((size + alignment - 1) / alignment) * alignment; }
    size_t alloc(size_t size);  // returns offset (best fit; grows the arena at the tail)
    void free(size_t offset, size_t size);
    size_t getPeak() const { return peak; }
    size_t getUsed() const { return used; }
    size_t numFreeBlocks() const { return freeByAddr.size(); }
    void reset();
};

// ---------------------------------------------------------------- execution schedule (fusion plan)
// The reference executes one kernel per operator in topological order and its GraphObj::optimize() is an
// empty hook (src/core/graph.cc:184-191).  Here the graph additionally derives an EXECUTION SCHEDULE: a list
// of steps, each one operator or a small group of operators that one fused kernel executes.  Alias / MatMul+Add /
// Silu*Mul steps are bit-identical to the unfused sequence; a MatMul group may use another split-K partition
// (fp32 summation order) and is held to the GEMM tolerance.  The memory planner takes tensor lifetimes from the schedule and the
// runtime dispatches it.  ITB_NO_FUSION=1 yields the 1:1 schedule.
struct ExecStep {
    enum Kind {
        Single,       // one operator, dispatched through the KernelRegistry
        Alias,        // Reshape / Flatten / Squeeze / Unsqueeze / Identity / size-1-only Transpose whose output
                      // shares the input's storage (no launch); falls back to the copy kernel if the planner
                      // gave them distinct storage
        MatMulGroup,  // 2..4 MatMuls sharing the activation operand (q/k/v, gate/up): one grouped launch
        MatMulAdd,    // MatMul -> Add(residual): residual added in the GEMM epilogue
        SiluMul,      // Silu -> Mul: one pass
        AttentionRope,    // RoPE(q), RoPE(k) -> [aliases] -> AttentionKVCache: RoPE applied inside the attention kernel
        AllReduceAddNorm, // AllReduceSum -> Add(residual) [-> RMSNorm]: one NVLink peer-memory kernel (else 3 ops)
        ConvBnAct,        // Conv -> BatchNorm -> [Add(residual)] -> [Relu]: the tail runs in the tensor-core GEMM epilogue
                          // (bit-identical to the separate kernels); shapes the GEMM does not take run one by one
        PrefillAttention  // Transpose(k) -> MatMul(q, .) -> [Div | Mul scalar] -> [Add mask] -> Softmax(-1) -> MatMul(., v): one wgmma
                          // kernel per (batch, head, 128-query tile) (kernels/attention_prefill.cu); ops in that order
    } kind = Single;
    OpVec ops;
    // NHWC domain (schedule.cc assignLayouts): bit 0 = the step's 4-D activation operands are stored [N, H, W, C], bit 1 = its
    // result is.  The tensors keep their logical NCHW dims; only Conv / Pool / same-shape Add / Relu steps carry these bits, and
    // graph inputs, outputs and every tensor some other operator reads stay NCHW.
    int layout = 0;
};

// ---------------------------------------------------------------- Graph
class GraphObj : public std::enable_shared_from_this<GraphObj> {
    Runtime runtime;
    TensorVec tensors;
    OpVec ops;
    bool sorted = true;
    uint64_t graphId, storageEpoch = 0;
    mutable uint64_t topologyEpoch = 0, seenFlagsEpoch = 0;
    Blob weightArena, activationArena;
    size_t weightBytes = 0, activationBytes = 0;
    bool weightsAllocated = false;

    void addOperatorAndConnect(const Operator &op);
    vector<ExecStep> schedule;
    uint64_t scheduleEpoch = ~0ull;

  public:
    // steps in execution order; rebuilt when the topology changes
    const vector<ExecStep> &getSchedule();
    explicit GraphObj(Runtime runtime);
    Runtime getRuntime() const { return runtime; }
    Tensor addTensor(Shape dim, DataType dtype = DataType::Float32);
    Tensor addTensor(const Tensor &tensor);
    const TensorVec &getTensors() const { return tensors; }
    const OpVec &getOperators() const { return ops; }
    Tensor getTensorByFuid(UidBaseType fuid) const;
    uint64_t getGraphId() const { return graphId; }
    uint64_t getTopologyEpoch() const {
        if (seenFlagsEpoch != TensorObj::flagsEpoch()) {  // a tensor flag changed somewhere: treat as a topology change
            seenFlagsEpoch = TensorObj::flagsEpoch();
            ++topologyEpoch;
        }
        return topologyEpoch;
    }
    uint64_t getStorageEpoch() const { return storageEpoch; }

    template <typename T, typename... Args> Ref<T> addOp(Args &&...args) {
        Ref<T> op = make_ref<T>(this, std::forward<Args>(args)...);
        addOperatorAndConnect(op);
        return op;
    }
    template <typename T, typename... Args> Ref<T> addOpWithOutputs(Args &&...args) {
        Ref<T> op = make_ref<T>(nullptr, std::forward<Args>(args)...);
        addOperatorAndConnect(op);
        return op;
    }

    void addOperator(const Operator &op) { addOperatorAndConnect(op); }
    bool topo_sort();
    void optimize() {}  // the reference's GraphObj::optimize is an empty switch (graph.cc:184-191)
    void shape_infer();
    void dataMalloc(bool useNaiveAllocator = false, size_t memPoolSize = 0);
    void validateMemory() const;
    size_t getWeightArenaBytes() const { return weightBytes; }
    size_t getActivationArenaBytes() const { return activationBytes; }
    TensorVec getInputs() const;
    TensorVec getOutputs() const;
    string toString() const;
};

template <typename T> string vecToString(const vector<T> &v) {
    std::ostringstream os;
    os << "[";
    for (size_t i = 0; i < v.size(); ++i) os << (i ? "," : "") << v[i];
    os << "]";
    return os.str();
}

// utils (reference src/utils/operator_utils.cc:6-44)
Shape infer_broadcast(const Shape &A, const Shape &B);
int get_real_axis(int axis, int rank);
HashType hashVector(const vector<int> &v);

}  // namespace infini
