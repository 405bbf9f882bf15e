// operators.h -- device-agnostic operator definitions for the hot path (shape / dtype inference +
// the typed getters the kernels read).  Same class names, constructor argument order and getters as
// the reference's include/operators/*.h so kernels and tests read identically; bodies are new.
//   MatmulObj ........ include/operators/matmul.h:9-72, src/operators/matmul.cc:26-49
//   ConvObj .......... include/operators/conv.h:111-150, src/operators/conv.cc:85-114
//   AttentionKVCacheObj include/operators/attention_kvcache.h:10-42
//   LayerNormObj ..... include/operators/layer_norm.h:5-29      RMSNormObj / RoPEObj: rms_norm.h, rope.h
//   UnaryObj family .. include/operators/unary.h:287-301         ElementWiseObj: element_wise.h:54-81
//   Transpose/Concat/Split/Gather/Reshape/Cast/Where/Expand/Reduce/Slice/Pad/Pooling/BatchNorm,
//   AllReduceBaseObj / AllGatherObj: the respective include/operators/*.h
#pragma once
#include "core.h"

namespace infini {

class MatmulObj : public OperatorObj {
    bool transA, transB;
    ActType act;
    mutable int b, m, n, k;
    string computeType;
    bool hasWScale = false;  // extension (SURVEY 8(f-4)): B holds FP8 E4M3 codes, the LAST input is its per-column f32 scale

  public:
    MatmulObj(GraphObj *graph, Tensor A, Tensor B, Tensor C, bool transA = false, bool transB = false,
              Tensor bias = nullptr, ActType act = ActType::None, string computeType = "default", Tensor wScale = nullptr);
    Tensor getWScale() const { return hasWScale ? inputs.back() : nullptr; }
    vector<DataType> inferDataType(const TensorVec &ins) const override { return {ins[0]->getDType()}; }
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    string toString() const override;
    vector<int> getWorkloadVector() const override;
    Tensor getBias() const { return inputs.size() > (hasWScale ? 3u : 2u) ? inputs[2] : nullptr; }
    ActType getAct() const { return act; }
    bool getTransA() const { return transA; }
    bool getTransB() const { return transB; }
    auto getBMNK() const { return std::tuple{b, m, n, k}; }
    int getB() const { return b; }
    int getM() const { return m; }
    int getN() const { return n; }
    int getK() const { return k; }
    string getComputeType() const { return computeType; }
};

// com.microsoft MatMulNBits with bits = 4 (extension; the reference has no quantised MatMul): Y[.., N] = A[.., K] . W,
// W[k, n] = (q[n, k] - z[n, k / bs]) * s[n, k / bs].  Inputs: A (f16 / bf16), B uint8 [N, K / bs, bs / 2] (column n's codes contiguous,
// even k in the low nibble), scales [N * K / bs] of A's dtype, optional zero_points uint8 [N * (K / bs) / 2] (nibble-packed, low
// nibble for even blocks; only when K / bs is even; absent: z = 8).  The layout is spelled out in it_b200.h (it_b200_matmul_nbits).
class MatMulNBitsObj : public OperatorObj {
    int K, N, bits, blockSize;

  public:
    // gIdx / bias: the operator's optional inputs 4 and 5, refused when present
    MatMulNBitsObj(GraphObj *graph, Tensor A, Tensor B, Tensor scales, Tensor zeroPoints, Tensor Y, int K, int N, int bits, int blockSize,
                   Tensor gIdx = nullptr, Tensor bias = nullptr);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    vector<DataType> inferDataType(const TensorVec &ins) const override { return {ins[0]->getDType()}; }
    vector<int> getOpAttrVector() const override { return {(int)type.underlying(), K, N, bits, blockSize, (int)inputs.size()}; }
    vector<int> getWorkloadVector() const override;
    Tensor getZeroPoints() const { return inputs.size() > 3 ? inputs[3] : nullptr; }
    int getK() const { return K; }
    int getN() const { return N; }
    int getBlockSize() const { return blockSize; }
};

class ConvObj : public OperatorObj {
    int ph, pw, sh, sw, dh, dw;
    ActType act;

  public:
    ConvObj(GraphObj *graph, Tensor input, Tensor weight, Tensor output, int ph, int pw, int sh = 1, int sw = 1,
            int dh = 1, int dw = 1, Tensor bias = nullptr, ActType act = ActType::None);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    // n, c, h, w, f, r, s (reference ConvBaseObj::getNCHWFRS, conv.h:111-119)
    auto getNCHWFRS() const {
        auto &x = inputs[0]->getDims();
        auto &w = inputs[1]->getDims();
        return std::tuple{x[0], x[1], x[2], x[3], w[0], w[2], w[3]};
    }
    auto getPadStrideDilation() const { return std::tuple{ph, pw, sh, sw, dh, dw}; }
    int getChannelPerGroup() const { return inputs[1]->getDims()[1]; }
    int getNumGroups() const { return inputs[0]->getDims()[1] / getChannelPerGroup(); }
    ActType getAct() const { return act; }
    vector<int> getWorkloadVector() const override;
};

// caches [B, Hkv, S_max, D], q [B, Hq, S, D], k / v [B, Hkv, S, D], Hq % Hkv == 0; output shaped as q.  Grouped-query
// attention (Hq = G Hkv, G > 1): query head i attends over KV head i / G, the order of HF's repeat_kv.
class AttentionKVCacheObj : public OperatorObj {
    bool perRowPositions;  // extension (SURVEY 8(f-3)): row b attends up to position_id[b]; false = the reference's element-0 rule
    int window;            // extension: sliding window, query at position P reads rows (P - window, P]; 0 = no window
    bool rolling;          // extension (needs a window): the caches are a ring, position P in row P mod S_max

  public:
    // k_scale / v_scale (extension): the caches hold FP8 E4M3 codes, element value e4m3(code) * scale[KV head]; f32 [Hkv]
    AttentionKVCacheObj(GraphObj *graph, Tensor input_k_cache, Tensor input_v_cache, Tensor input_q,
                        Tensor input_k, Tensor input_v, Tensor position_id, Tensor output_matmul,
                        bool perRowPositions = false, Tensor k_scale = nullptr, Tensor v_scale = nullptr, int window = 0,
                        bool rolling = false);
    bool getPerRowPositions() const { return perRowPositions; }
    int getWindow() const { return window; }
    bool getRolling() const { return rolling; }
    bool isFp8Cache() const { return inputs.size() == 8; }
    // window 0 keeps the attribute vector (and with it perf records and capture keys) of an unwindowed operator, and
    // rolling false that of a windowed one
    vector<int> getOpAttrVector() const override {
        if (!window) return {(int)type.underlying(), (int)perRowPositions};
        if (!rolling) return {(int)type.underlying(), (int)perRowPositions, window};
        return {(int)type.underlying(), (int)perRowPositions, window, 1};
    }
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    vector<DataType> inferDataType(const TensorVec &ins) const override { return {ins[2]->getDType()}; }
};

class SoftmaxObj : public OperatorObj {
    int axis;

  public:
    SoftmaxObj(GraphObj *graph, Tensor input, Tensor output, int axis);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override { return {{inputs[0]->getDims()}}; }
    int getAxis() const { return axis; }
    vector<int> getOpAttrVector() const override { return {(int)type.underlying(), axis}; }
};

class LayerNormObj : public OperatorObj {
    float eps;
    int axis, stash_type;

  public:
    LayerNormObj(GraphObj *graph, Tensor input, Tensor scale, Tensor output, Tensor bias = nullptr,
                 float eps = 1e-5, int axis = -1, int stash_type = 1);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override { return {{inputs[0]->getDims()}}; }
    Tensor getBias() const { return inputs.size() > 2 ? inputs[2] : nullptr; }
    float getEps() const { return eps; }
    int getAxis() const { return axis; }
    int getStashType() const { return stash_type; }
};

class RMSNormObj : public OperatorObj {
  public:
    RMSNormObj(GraphObj *graph, Tensor input, Tensor weight, Tensor output);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override { return {{inputs[0]->getDims()}}; }
};

class RoPEObj : public OperatorObj {
    int dimHead;  // extension: rotate-half over heads of this width; the reference fixes it at 128 (rope.cc:25)

  public:
    // invFreq (extension, optional): f32 [dimHead / 2]; column pair c of every head rotates by fp32(p x invFreq[c]) instead
    // of the reference's p x 10000^(-2c / dimHead)
    RoPEObj(GraphObj *graph, Tensor pos, Tensor input, Tensor output, int dimHead = 128, Tensor invFreq = nullptr);
    int getDimHead() const { return dimHead; }
    Tensor getInvFreq() const { return inputs.size() > 2 ? inputs[2] : nullptr; }
    vector<int> getOpAttrVector() const override { return {(int)type.underlying(), dimHead}; }
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    vector<DataType> inferDataType(const TensorVec &ins) const override { return {ins[1]->getDType()}; }
};

class UnaryObj : public OperatorObj {
  public:
    UnaryObj(OpType type, GraphObj *graph, Tensor input, Tensor output);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override { return {{inputs[0]->getDims()}}; }
};
#define DEFINE_UNARY_OBJ(prefix, type)                                                         \
    class prefix##Obj : public UnaryObj {                                                      \
      public:                                                                                  \
        prefix##Obj(GraphObj *graph, Tensor input, Tensor output) : UnaryObj(type, graph, input, output) {} \
    };
DEFINE_UNARY_OBJ(Relu, OpType::Relu)
DEFINE_UNARY_OBJ(Silu, OpType::Silu)
DEFINE_UNARY_OBJ(Gelu, OpType::Gelu)
DEFINE_UNARY_OBJ(Sigmoid, OpType::Sigmoid)
DEFINE_UNARY_OBJ(Tanh, OpType::Tanh)
DEFINE_UNARY_OBJ(HardSigmoid, OpType::HardSigmoid)
DEFINE_UNARY_OBJ(HardSwish, OpType::HardSwish)
DEFINE_UNARY_OBJ(Abs, OpType::Abs)
DEFINE_UNARY_OBJ(Sqrt, OpType::Sqrt)
DEFINE_UNARY_OBJ(Neg, OpType::Neg)
DEFINE_UNARY_OBJ(Erf, OpType::Erf)
DEFINE_UNARY_OBJ(Exp, OpType::Exp)
DEFINE_UNARY_OBJ(Identity, OpType::Identity)
// unary operators with a slope (reference include/operators/unary.h:50-62, 248-261)
class LeakyReluObj : public UnaryObj {
    float alphaValue;

  public:
    LeakyReluObj(GraphObj *graph, Tensor input, Tensor output, float alpha) : UnaryObj(OpType::LeakyRelu, graph, input, output), alphaValue(alpha) {}
    float getAlpha() const { return alphaValue; }
};
class EluObj : public UnaryObj {
  public:
    float alpha;
    EluObj(GraphObj *graph, Tensor input, Tensor output, float alpha) : UnaryObj(OpType::Elu, graph, input, output), alpha(alpha) {}
    float getAlpha() const { return alpha; }
};

class ElementWiseObj : public OperatorObj {
  public:
    ElementWiseObj(OpType type, GraphObj *graph, Tensor input0, Tensor input1, Tensor output);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    vector<DataType> inferDataType(const TensorVec &ins) const override;
};
#define DEFINE_ELEMENT_WISE_OBJ(prefix, type)                                                  \
    class prefix##Obj : public ElementWiseObj {                                                \
      public:                                                                                  \
        prefix##Obj(GraphObj *graph, Tensor a, Tensor b, Tensor c) : ElementWiseObj(type, graph, a, b, c) {} \
    };
DEFINE_ELEMENT_WISE_OBJ(Add, OpType::Add)
DEFINE_ELEMENT_WISE_OBJ(Sub, OpType::Sub)
DEFINE_ELEMENT_WISE_OBJ(Mul, OpType::Mul)
DEFINE_ELEMENT_WISE_OBJ(Div, OpType::Div)
DEFINE_ELEMENT_WISE_OBJ(Pow, OpType::Pow)
DEFINE_ELEMENT_WISE_OBJ(Maximum, OpType::Max)
DEFINE_ELEMENT_WISE_OBJ(Minimum, OpType::Min)
DEFINE_ELEMENT_WISE_OBJ(Less, OpType::Less)
DEFINE_ELEMENT_WISE_OBJ(Equal, OpType::Equal)
DEFINE_ELEMENT_WISE_OBJ(Greater, OpType::Greater)

class TransposeObj : public OperatorObj {
    vector<int> transposePermute;

  public:
    TransposeObj(GraphObj *graph, Tensor input, Tensor output, vector<int> permute);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    const vector<int> &getPermute() const { return transposePermute; }
    vector<int> getOpAttrVector() const override;
};

// DepthToSpace (reference include/operators/transpose.h:23-49, src/operators/transpose.cc:53-107): [N, C, H, W] ->
// [N, C / b^2, H b, W b]; executed as the rank-6 permutation the ONNX specification defines for each mode.
class DepthToSpaceObj : public OperatorObj {
    int blockSize, d2sMode;  // mode 0 = "DCR" (depth-column-row), 1 = "CRD"
    string modeString;
    mutable vector<int> reshapeDim, transposeDim, outDim;

  public:
    DepthToSpaceObj(GraphObj *graph, Tensor input, Tensor output, int blocksize, string mode);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    int getBlockSize() const { return blockSize; }
    int getMode() const { return d2sMode; }
    const string &getModeString() const { return modeString; }
    const vector<int> &getReshapeDim() const { return reshapeDim; }
    const vector<int> &getTransposeDim() const { return transposeDim; }
    const vector<int> &getOutDim() const { return outDim; }
    vector<int> getPermute() const { return d2sMode == 0 ? vector<int>{0, 3, 4, 1, 5, 2} : vector<int>{0, 1, 4, 2, 5, 3}; }
    vector<int> getOpAttrVector() const override { return {(int)type.underlying(), blockSize, d2sMode}; }
};

class ConcatObj : public OperatorObj {
    int dim;

  public:
    ConcatObj(GraphObj *graph, TensorVec inputs, Tensor output, int dim);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    int getDim() const { return dim; }
};

class SplitObj : public OperatorObj {
    int dim, num;
    vector<int> ratio;

  public:
    SplitObj(GraphObj *graph, Tensor input, std::optional<TensorVec> outputs, int dim, int num);
    SplitObj(GraphObj *graph, Tensor input, std::optional<TensorVec> outputs, int dim, const vector<int> &ratio);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    int getDim() const { return dim; }
    int numOutputs() const override { return num; }
};

class GatherObj : public OperatorObj {
    int axis;

  public:
    GatherObj(GraphObj *graph, Tensor input, Tensor indices, Tensor output, int axis);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    vector<DataType> inferDataType(const TensorVec &ins) const override { return {ins[0]->getDType()}; }
    int getAxis() const { return axis; }
};

// Reshape / Flatten / Identity / Squeeze / Unsqueeze: all lowered to a copy (reference reshape.cc:4-21)
class ReshapeObj : public OperatorObj {
    Shape dims;

  public:
    ReshapeObj(GraphObj *graph, Tensor input, Tensor output, Shape dims);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    Shape getShape() const { return dims; }
};
class FlattenObj : public OperatorObj {
    int axis;

  public:
    FlattenObj(GraphObj *graph, Tensor input, Tensor output, int axis);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    int getAxis() const { return axis; }
};
class SqueezeObj : public OperatorObj {
    vector<int> axes;

  public:
    SqueezeObj(GraphObj *graph, Tensor input, Tensor output, vector<int> axes);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
};
class UnsqueezeObj : public OperatorObj {
    vector<int> axes;

  public:
    UnsqueezeObj(GraphObj *graph, Tensor input, Tensor output, vector<int> axes);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
};

class CastObj : public OperatorObj {
    DataType to;

  public:
    CastObj(GraphObj *graph, Tensor input, Tensor output, DataType to);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override { return {{inputs[0]->getDims()}}; }
    vector<DataType> inferDataType(const TensorVec &) const override { return {to}; }
    DataType getOutputDataType() const { return to; }
};

class WhereObj : public OperatorObj {
  public:
    WhereObj(GraphObj *graph, Tensor inputX, Tensor inputY, Tensor condition, Tensor output);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
};

class ExpandObj : public OperatorObj {
    Shape dims;

  public:
    ExpandObj(GraphObj *graph, Tensor input, Tensor output, Shape dims);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    Shape getShape() const { return dims; }
};

class ReduceBaseObj : public OperatorObj {
    std::set<int> axes;
    bool keepDims;

  public:
    ReduceBaseObj(GraphObj *graph, OpType opType, Tensor input, Tensor output,
                  const std::optional<vector<int>> &axes, bool keepDims);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    bool isReduced(int idx) const { return axes.count(idx) > 0; }
    const std::set<int> &getAxes() const { return axes; }
    bool getKeepDims() const { return keepDims; }
};
class ReduceMeanObj : public ReduceBaseObj {
  public:
    ReduceMeanObj(GraphObj *graph, Tensor input, Tensor output, const std::optional<vector<int>> &axes,
                  bool keepDims = true)
        : ReduceBaseObj(graph, OpType::ReduceMean, input, output, axes, keepDims) {}
};
class ReduceSumObj : public ReduceBaseObj {
  public:
    ReduceSumObj(GraphObj *graph, Tensor input, Tensor output, const std::optional<vector<int>> &axes,
                 bool keepDims = true)
        : ReduceBaseObj(graph, OpType::ReduceSum, input, output, axes, keepDims) {}
};

class SliceObj : public OperatorObj {
    struct Range { int start, end, step; };
    vector<Range> axes;  // one per input dim

  public:
    SliceObj(GraphObj *graph, Tensor input, Tensor output, const vector<int> &starts, const vector<int> &ends,
             const std::optional<vector<int>> &axes, const std::optional<vector<int>> &steps);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    vector<int> getStarts() const;
    vector<int> getSteps() const;
};

class PadObj : public OperatorObj {
    vector<int> pads;  // [begin_0..begin_{r-1}, end_0..end_{r-1}]

  public:
    PadObj(GraphObj *graph, Tensor input, Tensor output, const vector<int> &pads,
           const std::optional<vector<int>> &axes);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    const vector<int> &getPads() const { return pads; }
};

class PoolingObj : public OperatorObj {
    int kh, kw, dh, dw, ph, pw, sh, sw, ceilMode;

  public:
    PoolingObj(GraphObj *graph, OpType optype, Tensor input, Tensor output, int kh, int kw, int dh, int dw, int ph,
               int pw, int sh, int sw, int ceilMode);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    auto getKDPS() const { return std::tuple{kh, kw, dh, dw, ph, pw, sh, sw}; }
    int getKh() const { return kh; }
    int getKw() const { return kw; }
    int getDh() const { return dh; }
    int getDw() const { return dw; }
    int getPh() const { return ph; }
    int getPw() const { return pw; }
    int getSh() const { return sh; }
    int getSw() const { return sw; }
    int getCeilMode() const { return ceilMode; }
};
class MaxPoolObj : public PoolingObj {
  public:
    MaxPoolObj(GraphObj *graph, Tensor input, Tensor output, int kh, int kw, int dh, int dw, int ph, int pw, int sh,
               int sw, int ceilMode)
        : PoolingObj(graph, OpType::MaxPool, input, output, kh, kw, dh, dw, ph, pw, sh, sw, ceilMode) {}
};
class AvgPoolObj : public PoolingObj {
  public:
    AvgPoolObj(GraphObj *graph, Tensor input, Tensor output, int kh, int kw, int dh, int dw, int ph, int pw, int sh,
               int sw, int ceilMode)
        : PoolingObj(graph, OpType::AveragePool, input, output, kh, kw, dh, dw, ph, pw, sh, sw, ceilMode) {}
};

class BatchNormObj : public OperatorObj {
    float momentum, eps;
    bool trainingMode;

  public:
    BatchNormObj(GraphObj *graph, Tensor input, Tensor output, Tensor mean, Tensor var, Tensor scale, Tensor bias,
                 float momentum = 0.9, float eps = 1e-5, bool trainingMode = false);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override { return {{inputs[0]->getDims()}}; }
    float getMomentum() const { return momentum; }
    float getEps() const { return eps; }
    bool getTrainingMode() const { return trainingMode; }
};

class AllReduceBaseObj : public OperatorObj {
  public:
    AllReduceBaseObj(GraphObj *graph, OpType opType, Tensor input, Tensor output);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override { return {{inputs[0]->getDims()}}; }
};
#define DEFINE_ALLREDUCE_OBJ(prefix, type)                                                     \
    class prefix##Obj : public AllReduceBaseObj {                                              \
      public:                                                                                  \
        prefix##Obj(GraphObj *graph, Tensor input, Tensor output) : AllReduceBaseObj(graph, type, input, output) {} \
    };
DEFINE_ALLREDUCE_OBJ(AllReduceSum, OpType::AllReduceSum)
DEFINE_ALLREDUCE_OBJ(AllReduceProd, OpType::AllReduceProd)
DEFINE_ALLREDUCE_OBJ(AllReduceMin, OpType::AllReduceMin)
DEFINE_ALLREDUCE_OBJ(AllReduceMax, OpType::AllReduceMax)
DEFINE_ALLREDUCE_OBJ(AllReduceAvg, OpType::AllReduceAvg)

class AllGatherObj : public OperatorObj {
    int world_size;

  public:
    AllGatherObj(GraphObj *graph, Tensor input, std::optional<TensorVec> outputs, int world_size);
    std::optional<vector<Shape>> inferShape(const TensorVec &inputs) override;
    int numOutputs() const override { return world_size; }
    int getWorldSize() const { return world_size; }
};

}  // namespace infini
