// core.cc -- Tensor / Operator / Graph / planner / registries (see core.h for the reference map).
#include "core.h"

#include <cctype>
#include <cstdlib>
#include <fstream>
#include <sstream>

#include <algorithm>
#include <atomic>
#include <numeric>
#include <unordered_set>

namespace infini {

const DataType DataType::Undefine(0), DataType::Float32(1), DataType::UInt8(2), DataType::Int8(3),
    DataType::UInt16(4), DataType::Int16(5), DataType::Int32(6), DataType::Int64(7), DataType::String(8),
    DataType::Bool(9), DataType::Float16(10), DataType::Double(11), DataType::UInt32(12), DataType::UInt64(13),
    DataType::BFloat16(16), DataType::Float8E4M3FN(17);

static const char *kOpNames[] = {
    "Unknown", "Abs", "Add", "AllGather", "AllReduceAvg", "AllReduceMax", "AllReduceMin", "AllReduceProd",
    "AllReduceSum", "AttentionKVCache", "AveragePool", "BatchNormalization", "Cast", "Concat", "Conv",
    "DepthToSpace", "Div", "Elu", "Equal", "Erf", "Exp", "Expand", "Flatten", "Gather", "Gelu", "Greater", "HardSigmoid",
    "HardSwish", "Identity", "LayerNormalization", "LeakyRelu", "Less", "MatMul", "Max", "MaxPool", "Min", "Mul", "Neg", "Pad",
    "Pow", "RMSNorm", "ReduceMean", "ReduceSum", "Relu", "Reshape", "RoPE", "Sigmoid", "Silu", "Slice", "Softmax",
    "Split", "Sqrt", "Squeeze", "Sub", "Tanh", "Transpose", "Unsqueeze", "Where", "MatMulNBits"};
static_assert(sizeof(kOpNames) / sizeof(kOpNames[0]) == OpType::NumOpTypes, "op name table out of sync");

const char *OpType::toString() const { return type < NumOpTypes ? kOpNames[type] : "Unknown"; }
OpType OpType::fromString(const string &s) {
    for (underlying_t i = 0; i < NumOpTypes; ++i)
        if (s == kOpNames[i]) return OpType(i);
    return OpType(Unknown);
}

static std::atomic<int> g_guid{0}, g_fuid{0};
static std::atomic<uint64_t> g_graph_id{0};

// ---------------------------------------------------------------- utils
Shape infer_broadcast(const Shape &A, const Shape &B) {
    if (A.empty() && B.empty()) return {};
    size_t r = std::max(A.size(), B.size());
    Shape ret(r);
    for (size_t i = 0; i < r; ++i) {
        int a = i < r - A.size() ? 1 : A[i - (r - A.size())];
        int b = i < r - B.size() ? 1 : B[i - (r - B.size())];
        IT_ASSERT(a == b || a == 1 || b == 1, "shapes are not broadcastable");
        ret[i] = a == 1 ? b : a;  // keeps 0-sized dims
    }
    return ret;
}
int get_real_axis(int axis, int rank) {
    IT_ASSERT(rank >= 1);
    IT_ASSERT(axis >= -rank && axis <= rank - 1, "axis out of range");
    return axis < 0 ? axis + rank : axis;
}
HashType hashVector(const vector<int> &v) {
    HashType h = 1469598103934665603ull;
    for (int x : v) {
        h ^= (HashType)(uint32_t)x;
        h *= 1099511628211ull;
    }
    return h;
}

// ---------------------------------------------------------------- Blob / Tensor
BlobObj::~BlobObj() {
    if (!owner && ptr && runtime) runtime->dealloc(ptr);  // only arena roots free (exactly once)
}

TensorObj::TensorObj(Shape shape, DataType dtype, Runtime runtime)
    : shape(std::move(shape)), dtype(dtype), runtime(std::move(runtime)), guid(++g_guid), fuid(++g_fuid) {
    for (int d : this->shape) IT_ASSERT(d >= 0, "negative dimension");
}
Shape TensorObj::getStride() const {
    Shape st(shape.size());
    int acc = 1;
    for (int i = (int)shape.size() - 1; i >= 0; --i) {
        st[i] = acc;
        acc *= shape[i];
    }
    return st;
}
size_t TensorObj::size() const {
    size_t n = 1;
    for (int d : shape) n *= (size_t)d;
    return n;
}
void TensorObj::dataMalloc() {
    if (data) return;
    size_t b = std::max<size_t>(getBytes(), 1);
    data = make_ref<BlobObj>(runtime, runtime->alloc(b), b);
}
void TensorObj::copyin(const void *host, size_t bytes) {
    IT_ASSERT(bytes == getBytes(), "copyin: size mismatch");
    if (bytes) runtime->copyBlobFromCPU(getRawDataPtr<void *>(), host, bytes);
}
void TensorObj::copyout(void *host, size_t bytes) const {
    IT_ASSERT(bytes == getBytes(), "copyout: size mismatch");
    if (bytes) runtime->copyBlobToCPU(host, getRawDataPtr<void *>(), bytes);
}
OpVec TensorObj::getTargets() const {
    OpVec r;
    for (auto &w : targets)
        if (auto p = w.lock()) r.push_back(p);
    return r;
}
string TensorObj::toString() const {
    return "Tensor " + std::to_string(guid) + ", Fuid " + std::to_string(fuid) + ", shape " + vecToString(shape) +
           ", dtype " + dtype.toString();
}

// ---------------------------------------------------------------- Operator
OperatorObj::OperatorObj(OpType type, TensorVec inputs, TensorVec outputs)
    : type(type), inputs(std::move(inputs)), outputs(std::move(outputs)), guid(++g_guid) {
    for (auto &t : this->inputs) IT_ASSERT(t, "operator input is null");
}
vector<DataType> OperatorObj::inferDataType(const TensorVec &ins) const {
    return vector<DataType>(numOutputs(), ins[0]->getDType());
}
string OperatorObj::toString() const {
    std::ostringstream os;
    os << type.toString() << "[" << guid << "](";
    for (auto &t : inputs) os << "i" << t->getGuid() << vecToString(t->getDims()) << ",";
    for (auto &t : outputs)
        if (t) os << "o" << t->getGuid() << vecToString(t->getDims()) << ",";
    os << ")";
    return os.str();
}
vector<int> OperatorObj::getWorkloadVector() const {
    vector<int> r{(int)type.underlying()};
    for (auto &t : inputs) r.insert(r.end(), t->getDims().begin(), t->getDims().end());
    return r;
}
OpPerfKey OperatorObj::getOpPerfKey() const {
    auto w = getWorkloadVector();
    return OpPerfKey{hashVector(w), type.underlying(), std::move(w)};
}
// validate inputs, infer output shapes/dtypes, create (or check) outputs -- reference src/core/operator.cc:59-80
bool OperatorObj::checkValid(GraphObj *graph) {
    auto shapes = inferShape(inputs);
    if (!shapes) return false;
    auto dts = inferDataType(inputs);
    IT_ASSERT(shapes->size() == outputs.size(), "inferShape/outputs count mismatch");
    for (size_t i = 0; i < outputs.size(); ++i) {
        if (outputs[i]) {
            IT_ASSERT((*shapes)[i] == outputs[i]->getDims(),
                      string("output shape mismatch in ") + type.toString() + ": inferred " +
                          vecToString((*shapes)[i]) + " given " + vecToString(outputs[i]->getDims()));
        } else {
            IT_ASSERT(graph != nullptr, "operator built without a graph must be given its outputs");
            outputs[i] = graph->addTensor((*shapes)[i], dts[i]);
        }
    }
    return true;
}
OpVec OperatorObj::getPredecessors() const {
    OpVec r;
    for (auto &w : predecessors)
        if (auto p = w.lock()) r.push_back(p);
    return r;
}
OpVec OperatorObj::getSuccessors() const {
    OpVec r;
    for (auto &w : successors)
        if (auto p = w.lock()) r.push_back(p);
    return r;
}

// ---------------------------------------------------------------- registries
KernelRegistry::~KernelRegistry() {
    for (auto &kv : kernels) delete kv.second.first;
}
KernelRegistry &KernelRegistry::getInstance() {
    static KernelRegistry inst;
    return inst;
}
bool KernelRegistry::registerKernel(const KernelAttrs &key, Kernel *kernel, string name) {
    IT_ASSERT(kernels.find(key) == kernels.end(), "Kernel already registered: " + name);
    kernels.emplace(key, std::pair<Kernel *const, const string>(kernel, std::move(name)));
    ++nKernels;
    return true;
}
Kernel *KernelRegistry::getKernel(const KernelAttrs &attrs) const {
    auto it = kernels.find(attrs);
    IT_ASSERT(it != kernels.end(), string("Kernel not found for ") + OpType(attrs.op).toString() + " on device " +
                                       std::to_string((int)attrs.device) + " (no CPU fallback exists)");
    return it->second.first;
}
const string &KernelRegistry::getKernelName(const KernelAttrs &attrs) const {
    auto it = kernels.find(attrs);
    IT_ASSERT(it != kernels.end(), "Kernel not found");
    return it->second.second;
}
PerfEngine &PerfEngine::getInstance() {
    static PerfEngine inst;
    return inst;
}
std::optional<PerfRecord> PerfEngine::getPerfData(const Key &key) const {
    auto it = data.find(key);
    if (it == data.end()) return std::nullopt;
    return it->second;
}
void PerfEngine::setPerfData(const Key &key, PerfRecord record) {
    IT_ASSERT(data.find(key) == data.end(), "Perf data already exist");
    data.emplace(key, std::move(record));
}

// ---- PerfEngine <-> JSON (a tiny reader for exactly the value kinds that layout uses: arrays, objects, numbers)
namespace {
struct JVal {
    enum Kind { Num, Arr, Obj } kind = Num;
    double num = 0;
    unsigned long long u64 = 0;  // exact value of a non-negative integer literal (hashes are 64-bit)
    vector<JVal> arr;
    vector<std::pair<string, JVal>> obj;
    const JVal &at(const string &k) const {
        for (auto &kv : obj)
            if (kv.first == k) return kv.second;
        throw Exception("perf-engine json: missing key '" + k + "'");
    }
};
struct JParser {
    const string &s;
    size_t i = 0;
    explicit JParser(const string &text) : s(text) {}
    void ws() {
        while (i < s.size() && (s[i] == ' ' || s[i] == '\n' || s[i] == '\t' || s[i] == '\r')) ++i;
    }
    void expect(char c) {
        ws();
        IT_ASSERT(i < s.size() && s[i] == c, string("perf-engine json: expected '") + c + "' at offset " + std::to_string(i));
        ++i;
    }
    bool peek(char c) {
        ws();
        return i < s.size() && s[i] == c;
    }
    string str() {
        expect('"');
        size_t b = i;
        while (i < s.size() && s[i] != '"') ++i;
        IT_ASSERT(i < s.size(), "perf-engine json: unterminated string");
        return s.substr(b, i++ - b);
    }
    JVal value() {
        ws();
        JVal v;
        if (peek('[')) {
            v.kind = JVal::Arr;
            ++i;
            if (peek(']')) { ++i; return v; }
            do v.arr.push_back(value()); while (peek(',') && ++i);
            expect(']');
        } else if (peek('{')) {
            v.kind = JVal::Obj;
            ++i;
            if (peek('}')) { ++i; return v; }
            do {
                string k = str();
                expect(':');
                v.obj.emplace_back(std::move(k), value());
            } while (peek(',') && ++i);
            expect('}');
        } else {
            size_t b = i;
            while (i < s.size() && (std::isdigit((unsigned char)s[i]) || s[i] == '-' || s[i] == '+' || s[i] == '.' || s[i] == 'e' || s[i] == 'E')) ++i;
            IT_ASSERT(i > b, "perf-engine json: unexpected character at offset " + std::to_string(b));
            const string tok = s.substr(b, i - b);
            v.num = std::strtod(tok.c_str(), nullptr);
            if (tok.find_first_of(".eE-") == string::npos) v.u64 = std::strtoull(tok.c_str(), nullptr, 10);
            else v.u64 = (unsigned long long)v.num;
        }
        return v;
    }
};
}  // namespace

void PerfEngine::savePerfEngineData(const string &path) const {
    std::ofstream out(path, std::ios::out | std::ios::trunc | std::ios::binary);
    IT_ASSERT(out.good(), "cannot write " + path);
    out << "{\"data\":[";
    bool first = true;
    for (auto &[key, rec] : data) {
        const auto &[attrs, perfKey] = key;
        out << (first ? "" : ",") << "[[[" << (int)attrs.device << "," << (long long)attrs.op << "],{\"attrs\":[";
        for (size_t k = 0; k < perfKey.attrs.size(); ++k) out << (k ? "," : "") << perfKey.attrs[k];
        out << "],\"hashType\":" << (unsigned long long)perfKey.hash << ",\"opType\":" << (long long)perfKey.opType << "}],{\"data\":";
        out.precision(17);
        out << rec->time << ",\"type\":" << rec->type();
        if (auto mr = std::dynamic_pointer_cast<MatmulPerfRecordObj>(rec)) out << ",\"impl\":" << mr->impl << ",\"nb\":" << mr->nb;
        out << "}]";
        first = false;
    }
    out << "]}" << std::endl;
}

void PerfEngine::loadPerfEngineData(const string &path) {
    std::ifstream in(path, std::ios::in | std::ios::binary);
    IT_ASSERT(in.good(), "cannot read " + path);
    std::stringstream ss;
    ss << in.rdbuf();
    const string text = ss.str();
    JParser p(text);
    JVal root = p.value();
    std::map<Key, PerfRecord> fresh;
    for (auto &entry : root.at("data").arr) {
        IT_ASSERT(entry.arr.size() == 2 && entry.arr[0].arr.size() == 2 && entry.arr[0].arr[0].arr.size() == 2, "perf-engine json: bad entry");
        const JVal &ka = entry.arr[0].arr[0], &pk = entry.arr[0].arr[1], &rec = entry.arr[1];
        OpPerfKey perfKey;
        perfKey.hash = (HashType)pk.at("hashType").u64;
        perfKey.opType = (OpType::underlying_t)pk.at("opType").num;
        for (auto &a : pk.at("attrs").arr) perfKey.attrs.push_back((int)a.num);
        const int rtype = (int)rec.at("type").num;
        IT_ASSERT(rtype == 0 || rtype == 1, "perf-engine json: record type " + std::to_string(rtype) + " is not one of this runtime's (0 plain, 1 MatMul)");
        PerfRecord r;
        if (rtype == 1) {
            auto mr = make_ref<MatmulPerfRecordObj>();
            mr->impl = (int)rec.at("impl").num;
            mr->nb = (int)rec.at("nb").num;
            r = mr;
        } else {
            r = make_ref<PerfRecordObj>();
        }
        r->time = rec.at("data").num;
        fresh[Key{KernelAttrs{(Device)(int)ka.arr[0].num, (OpType::underlying_t)ka.arr[1].num}, perfKey}] = r;
    }
    data = std::move(fresh);
}

double RuntimeObj::getPerfTime(const Graph &graph) const {
    double total = 0;
    auto &pe = PerfEngine::getInstance();
    for (auto &op : graph->getOperators()) {
        PerfEngine::Key key{KernelAttrs{device, op->getOpType().underlying()}, op->getOpPerfKey()};
        auto rec = pe.getPerfData(key);
        if (rec) total += (*rec)->time;
    }
    return total;
}

// ---------------------------------------------------------------- LazyAllocator
void LazyAllocator::insertFree(size_t off, size_t size) {
    freeByAddr[off] = size;
    freeBySize.insert({size, off});
}
void LazyAllocator::eraseFree(size_t off, size_t size) {
    freeByAddr.erase(off);
    freeBySize.erase({size, off});
}
size_t LazyAllocator::alloc(size_t size) {
    size = getAlignedSize(std::max<size_t>(size, 1));
    auto it = freeBySize.lower_bound({size, 0});
    size_t off;
    if (it != freeBySize.end()) {  // best fit
        size_t bsz = it->first;
        off = it->second;
        eraseFree(off, bsz);
        if (bsz > size) insertFree(off + size, bsz - size);
    } else {
        // grow at the tail; if the last free block touches the tail, extend it
        off = peak;
        auto last = freeByAddr.empty() ? freeByAddr.end() : std::prev(freeByAddr.end());
        if (last != freeByAddr.end() && last->first + last->second == peak) {
            off = last->first;
            eraseFree(last->first, last->second);
        }
        peak = off + size;
    }
    used += size;
    return off;
}
void LazyAllocator::free(size_t offset, size_t size) {
    size = getAlignedSize(std::max<size_t>(size, 1));
    used -= size;
    auto next = freeByAddr.lower_bound(offset);
    if (next != freeByAddr.end() && offset + size == next->first) {
        size += next->second;
        eraseFree(next->first, next->second);
    }
    auto prev = freeByAddr.lower_bound(offset);
    if (prev != freeByAddr.begin()) {
        --prev;
        if (prev->first + prev->second == offset) {
            offset = prev->first;
            size += prev->second;
            eraseFree(prev->first, prev->second);
        }
    }
    insertFree(offset, size);
}
void LazyAllocator::reset() {
    used = peak = 0;
    freeByAddr.clear();
    freeBySize.clear();
}

// ---------------------------------------------------------------- Graph
GraphObj::GraphObj(Runtime runtime) : runtime(std::move(runtime)), graphId(++g_graph_id) {}

Tensor GraphObj::addTensor(Shape dim, DataType dtype) {
    auto t = make_ref<TensorObj>(std::move(dim), dtype, runtime);
    tensors.push_back(t);
    return t;
}
Tensor GraphObj::addTensor(const Tensor &tensor) {
    IT_ASSERT(tensor->getRuntime() == runtime, "tensor belongs to another runtime");
    tensors.push_back(tensor);
    return tensor;
}
Tensor GraphObj::getTensorByFuid(UidBaseType fuid) const {
    for (auto &t : tensors)
        if (t->getFuid() == fuid) return t;
    return nullptr;
}
void GraphObj::addOperatorAndConnect(const Operator &op) {
    sorted = false;
    ++topologyEpoch;
    ops.push_back(op);
    for (auto &in : op->getInputs()) {
        in->targets.push_back(op);
        if (auto pred = in->getSource()) {
            pred->successors.push_back(op);
            op->predecessors.push_back(pred);
        }
    }
    for (auto &out : op->getOutputs()) {
        out->source = op;
        for (auto &succ : out->getTargets()) {
            succ->predecessors.push_back(op);
            op->successors.push_back(succ);
        }
    }
}
bool GraphObj::topo_sort() {
    if (sorted) return true;
    OpVec order;
    std::set<OperatorObj *> done;
    order.reserve(ops.size());
    while (order.size() < ops.size()) {
        bool progressed = false;
        for (auto &op : ops) {
            if (done.count(op.get())) continue;
            bool ready = true;
            for (auto &in : op->getInputs()) {
                auto src = in->getSource();
                if (src && !done.count(src.get())) {
                    ready = false;
                    break;
                }
            }
            if (ready) {
                order.push_back(op);
                done.insert(op.get());
                progressed = true;
            }
        }
        if (!progressed) return false;  // cycle
    }
    ops = std::move(order);
    sorted = true;
    return true;
}
void GraphObj::shape_infer() {
    IT_ASSERT(topo_sort(), "graph has a cycle");
    for (auto &op : ops) {
        auto shapes = op->inferShape();
        IT_ASSERT(shapes.has_value(), "shape inference failed for " + op->toString());
        IT_ASSERT(shapes->size() == op->getOutputs().size());
        for (size_t i = 0; i < shapes->size(); ++i)
            if ((*shapes)[i] != op->getOutput(i)->getDims()) {
                op->getOutput(i)->setShape((*shapes)[i]);
                ++topologyEpoch;
            }
    }
}
TensorVec GraphObj::getInputs() const {
    TensorVec r;
    for (auto &t : tensors)
        if (!t->getSource() && !t->isWeight()) r.push_back(t);
    return r;
}
TensorVec GraphObj::getOutputs() const {
    TensorVec r;
    for (auto &t : tensors)
        if (!t->hasTarget() || t->isOutput()) r.push_back(t);
    return r;
}

// Offline memory plan (semantics of reference src/core/graph.cc:341-576):
//   weights      -> one weight arena, allocated once and kept across re-plans
//   inputs/outputs -> pinned for the life of the plan
//   activations  -> alloc at the producing op, free after the last consuming op (refcounts, topological
//                   order), best-fit offsets inside one activation arena; 256 B aligned;
//   each arena is ONE runtime->alloc.  Transactional: nothing visible changes if an allocation throws.
void GraphObj::dataMalloc(bool useNaiveAllocator, size_t memPoolSize) {
    (void)memPoolSize;
    IT_ASSERT(topo_sort(), "graph has a cycle");
    const size_t align = runtime->getAlignment();
    LazyAllocator wAlloc(align), aAlloc(align);
    std::unordered_map<TensorObj *, size_t> wOff, aOff;

    bool needWeights = !weightsAllocated;
    for (auto &t : tensors)
        if (t->isWeight()) {
            if (!t->hasData()) needWeights = true;
        }
    if (needWeights)
        for (auto &t : tensors)
            if (t->isWeight()) wOff[t.get()] = wAlloc.alloc(t->getBytes());

    // lifetimes follow the EXECUTION SCHEDULE (fused steps allocate all member outputs when the step runs and
    // release inputs after it); Alias steps make the output share its input's storage (one refcounted root)
    const auto &sched = getSchedule();
    std::unordered_map<TensorObj *, TensorObj *> parent;
    auto root = [&](TensorObj *t) {
        while (true) {
            auto it = parent.find(t);
            if (it == parent.end()) return t;
            t = it->second;
        }
    };
    if (!useNaiveAllocator) {
        for (auto &st : sched) {
            if (st.kind != ExecStep::Alias) continue;
            auto in = st.ops[0]->getInputs(0), out = st.ops[0]->getOutput();
            if (!in->isWeight() && !out->isWeight()) parent[out.get()] = in.get();
        }
    }
    std::unordered_map<TensorObj *, int> refs;
    std::unordered_set<TensorObj *> pinnedRoots;
    auto pinned = [&](const Tensor &t) { return !t->getSource() || !t->hasTarget() || t->isOutput() || t->isInput(); };
    for (auto &t : tensors) {
        if (t->isWeight()) continue;
        TensorObj *r = root(t.get());
        refs[r] += (int)t->getTargets().size();
        if (pinned(t)) pinnedRoots.insert(r);
    }
    for (auto &t : tensors) {
        if (t->isWeight() || root(t.get()) != t.get()) continue;
        if (pinnedRoots.count(t.get()) || useNaiveAllocator) aOff[t.get()] = aAlloc.alloc(t->getBytes());
    }
    if (!useNaiveAllocator) {
        for (auto &st : sched) {
            for (auto &op : st.ops)
                for (auto &out : op->getOutputs()) {
                    if (out->isWeight()) continue;
                    TensorObj *r = root(out.get());
                    if (!aOff.count(r)) aOff[r] = aAlloc.alloc(r->getBytes());
                }
            for (auto &op : st.ops)
                for (auto &in : op->getInputs()) {
                    if (in->isWeight()) continue;
                    TensorObj *r = root(in.get());
                    if (pinnedRoots.count(r)) continue;
                    if (--refs[r] == 0) aAlloc.free(aOff[r], r->getBytes());
                }
        }
    }
    // every aliased tensor takes its root's offset
    for (auto &t : tensors)
        if (!t->isWeight() && root(t.get()) != t.get()) aOff[t.get()] = aOff.at(root(t.get()));

    // commit: allocate the arenas first (may throw), then bind views
    Blob newW = weightArena, newA;
    if (needWeights) {
        size_t wb = std::max<size_t>(wAlloc.getPeak(), align);
        newW = make_ref<BlobObj>(runtime, runtime->alloc(wb), wb);
        weightBytes = wAlloc.getPeak();
    }
    size_t ab = std::max<size_t>(aAlloc.getPeak(), align);
    newA = make_ref<BlobObj>(runtime, runtime->alloc(ab), ab);
    activationBytes = aAlloc.getPeak();

    if (needWeights) {
        for (auto &kv : wOff) {
            TensorObj *t = kv.first;
            // weights that already hold data (set before a re-plan) keep their bytes
            auto view = make_ref<BlobObj>(runtime, newW->getPtr<char *>() + kv.second, t->getBytes(), newW);
            if (t->hasData() && t->getBytes())
                runtime->copyBlobInsideRuntime(view->getPtr<void *>(), t->getRawDataPtr<void *>(), t->getBytes());
            t->setDataBlob(view);
        }
        weightArena = newW;
        weightsAllocated = true;
    }
    for (auto &kv : aOff) {
        TensorObj *t = kv.first;
        auto view = make_ref<BlobObj>(runtime, newA->getPtr<char *>() + kv.second, t->getBytes(), newA);
        // graph inputs keep previously copied-in contents across a re-plan
        if (t->hasData() && !t->getSource() && t->getBytes() && t->getDataBlob()->getBytes() == t->getBytes())
            runtime->copyBlobInsideRuntime(view->getPtr<void *>(), t->getRawDataPtr<void *>(), t->getBytes());
        t->setDataBlob(view);
    }
    activationArena = newA;
    ++storageEpoch;
}

void GraphObj::validateMemory() const {
    for (auto &t : tensors) IT_ASSERT(t->hasData(), "tensor without storage: " + t->toString());
}

string GraphObj::toString() const {
    std::ostringstream os;
    os << "Graph " << graphId << ": " << tensors.size() << " tensors, " << ops.size() << " operators\n";
    for (auto &op : ops) os << "  " << op->toString() << "\n";
    return os.str();
}

}  // namespace infini
