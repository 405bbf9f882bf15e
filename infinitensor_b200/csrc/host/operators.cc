// operators.cc -- shape rules of the hot-path operators (see operators.h for the reference map).
#include "operators.h"

#include <algorithm>
#include <numeric>

namespace infini {

// ---------------------------------------------------------------- MatMul (src/operators/matmul.cc:26-49)
static TensorVec matmulInputs(Tensor A, Tensor B, Tensor bias, Tensor wScale) {
    TensorVec v{A, B};
    if (bias) v.push_back(bias);
    if (wScale) v.push_back(wScale);
    return v;
}
MatmulObj::MatmulObj(GraphObj *graph, Tensor A, Tensor B, Tensor C, bool transA, bool transB, Tensor bias,
                     ActType act, string computeType, Tensor wScale)
    : OperatorObj(OpType::MatMul, matmulInputs(A, B, bias, wScale), {C}), transA(transA),
      transB(transB), act(act), b(1), m(0), n(0), k(0), computeType(std::move(computeType)), hasWScale(wScale != nullptr) {
    if (wScale) {
        IT_ASSERT(B->getDType() == DataType::Float8E4M3FN && wScale->getDType() == DataType::Float32,
                  "MatMul: a weight scale goes with an FP8 E4M3 weight and is f32");
        IT_ASSERT(B->getRank() == 2 && !transB && (int)wScale->size() == B->getDims()[1], "MatMul: one scale per output column of a [K, N] weight");
    } else {
        IT_ASSERT(B->getDType() != DataType::Float8E4M3FN, "MatMul: an FP8 weight needs its scale");
    }
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> MatmulObj::inferShape(const TensorVec &ins) {
    auto &sa = ins[0]->getDims();
    auto &sb = ins[1]->getDims();
    int ra = (int)sa.size(), rb = (int)sb.size();
    IT_ASSERT(ra >= 2 && rb >= 2, "MatMul needs rank >= 2 operands");
    Shape ba(sa.begin(), sa.end() - 2), bb(sb.begin(), sb.end() - 2);
    Shape ret = infer_broadcast(ba, bb);
    b = ret.empty() ? 1 : std::accumulate(ret.begin(), ret.end(), 1, std::multiplies<int>());
    int kA = transA ? sa[ra - 2] : sa[ra - 1];
    int kB = transB ? sb[rb - 1] : sb[rb - 2];
    IT_ASSERT(kA == kB, "MatMul: inner dimensions differ");
    m = transA ? sa[ra - 1] : sa[ra - 2];
    n = transB ? sb[rb - 2] : sb[rb - 1];
    k = kA;
    ret.push_back(m);
    ret.push_back(n);
    return {{ret}};
}
string MatmulObj::toString() const {
    std::ostringstream os;
    os << "Matmul([" << (transA ? "A^T" : "A") << "," << (transB ? "B^T" : "B") << ",act=" << (int)act
       << "],A=" << inputs[0]->getGuid() << ",B=" << inputs[1]->getGuid() << ",C=" << outputs[0]->getGuid()
       << ",bmnk=[" << b << "," << m << "," << n << "," << k << "]),computeType=" << computeType;
    return os.str();
}
vector<int> MatmulObj::getWorkloadVector() const {
    return {(int)type.underlying(), b, m, n, k, transA, transB, (int)act, inputs[0]->getDTypeIndex()};
}

// ---------------------------------------------------------------- MatMulNBits (extension)
static TensorVec nbitsInputs(Tensor A, Tensor B, Tensor scales, Tensor zp) {
    TensorVec v{A, B, scales};
    if (zp) v.push_back(zp);
    return v;
}
MatMulNBitsObj::MatMulNBitsObj(GraphObj *graph, Tensor A, Tensor B, Tensor scales, Tensor zeroPoints, Tensor Y, int K, int N, int bits,
                               int blockSize, Tensor gIdx, Tensor bias)
    : OperatorObj(OpType::MatMulNBits, nbitsInputs(A, B, scales, zeroPoints), {Y}), K(K), N(N), bits(bits), blockSize(blockSize) {
    IT_ASSERT(bits == 4, "MatMulNBits: bits = " + std::to_string(bits) + "; only 4-bit weights are supported");
    IT_ASSERT(blockSize == 32 || blockSize == 64 || blockSize == 128,
              "MatMulNBits: block_size = " + std::to_string(blockSize) + " is not 32, 64 or 128");
    IT_ASSERT(K > 0 && K % blockSize == 0,
              "MatMulNBits: K = " + std::to_string(K) + " is not a positive multiple of block_size " + std::to_string(blockSize));
    IT_ASSERT(N > 0 && N % 16 == 0, "MatMulNBits: N = " + std::to_string(N) + " is not a positive multiple of 16");
    IT_ASSERT(!gIdx, "MatMulNBits: the g_idx input (act-order) is not supported");
    IT_ASSERT(!bias, "MatMulNBits: the bias input is not supported");
    const auto dt = A->getDType();
    IT_ASSERT(dt != DataType::Float32, "MatMulNBits: fp32 activations are not supported (f16 / bf16 only)");
    IT_ASSERT(dt == DataType::Float16 || dt == DataType::BFloat16, "MatMulNBits: A must be f16 or bf16, not " + dt.toString());
    const int nblk = K / blockSize;
    IT_ASSERT(B->getDType() == DataType::UInt8 && B->getDims() == Shape({N, nblk, blockSize / 2}),
              "MatMulNBits: B must be uint8 [N, K / block_size, block_size / 2] = " + vecToString(Shape({N, nblk, blockSize / 2})) +
                  ", got " + B->getDType().toString() + " " + vecToString(B->getDims()));
    IT_ASSERT(scales->getDType() == dt && (int64_t)scales->size() == (int64_t)N * nblk,
              "MatMulNBits: scales must hold N * K / block_size = " + std::to_string((int64_t)N * nblk) + " values of A's dtype");
    if (zeroPoints) {
        IT_ASSERT(nblk % 2 == 0, "MatMulNBits: zero points need an even number of blocks per column (K / block_size = " +
                                     std::to_string(nblk) + ")");
        IT_ASSERT(zeroPoints->getDType() == DataType::UInt8 && (int64_t)zeroPoints->size() == (int64_t)N * nblk / 2,
                  "MatMulNBits: zero_points must be uint8 with N * (K / block_size) / 2 = " + std::to_string((int64_t)N * nblk / 2) +
                      " packed bytes");
    }
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> MatMulNBitsObj::inferShape(const TensorVec &ins) {
    Shape s = ins[0]->getDims();
    IT_ASSERT(!s.empty() && s.back() == K, "MatMulNBits: the last dimension of A must be K = " + std::to_string(K));
    s.back() = N;
    return {{s}};
}
vector<int> MatMulNBitsObj::getWorkloadVector() const {
    int rows = (int)(inputs[0]->size() / K);
    return {(int)type.underlying(), rows, N, K, blockSize, (int)inputs.size(), inputs[0]->getDTypeIndex()};
}

// ---------------------------------------------------------------- Conv (src/operators/conv.cc:85-114)
ConvObj::ConvObj(GraphObj *graph, Tensor input, Tensor weight, Tensor output, int ph, int pw, int sh, int sw,
                 int dh, int dw, Tensor bias, ActType act)
    : OperatorObj(OpType::Conv, {input, weight}, {output}), ph(ph), pw(pw), sh(sh), sw(sw), dh(dh), dw(dw),
      act(act) {
    IT_ASSERT(bias == nullptr, "Conv bias is lowered to Reshape+Add by the frontend (reference conv.cc:68-69)");
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> ConvObj::inferShape(const TensorVec &ins) {
    auto &x = ins[0]->getDims();
    auto &w = ins[1]->getDims();
    IT_ASSERT(x.size() == 4 && w.size() == 4, "Conv expects NCHW input and FCRS weight");
    IT_ASSERT(w[1] > 0 && x[1] % w[1] == 0, "Conv: input channels not divisible by weight channels");
    int groups = x[1] / w[1];
    IT_ASSERT(w[0] % groups == 0, "Conv: output channels not divisible by groups");
    int oh = (x[2] + 2 * ph - dh * (w[2] - 1) - 1) / sh + 1;
    int ow = (x[3] + 2 * pw - dw * (w[3] - 1) - 1) / sw + 1;
    return {{{x[0], w[0], oh, ow}}};
}
vector<int> ConvObj::getWorkloadVector() const {
    auto [n, c, h, w, f, r, s] = getNCHWFRS();
    return {(int)type.underlying(), n, c, h, w, f, r, s, ph, pw, sh, sw, dh, dw, inputs[0]->getDTypeIndex()};
}

// ---------------------------------------------------------------- AttentionKVCache (attention_kvcache.cc:5-27)
static TensorVec attentionInputs(TensorVec v, Tensor kScale, Tensor vScale) {
    IT_ASSERT(!kScale == !vScale, "AttentionKVCache: k_scale and v_scale go together");
    if (kScale) {
        v.push_back(kScale);
        v.push_back(vScale);
    }
    return v;
}
AttentionKVCacheObj::AttentionKVCacheObj(GraphObj *graph, Tensor input_k_cache, Tensor input_v_cache,
                                         Tensor input_q, Tensor input_k, Tensor input_v, Tensor position_id,
                                         Tensor output_matmul, bool perRowPositions, Tensor k_scale, Tensor v_scale, int window,
                                         bool rolling)
    : OperatorObj(OpType::AttentionKVCache,
                  attentionInputs({input_k_cache, input_v_cache, input_q, input_k, input_v, position_id}, k_scale, v_scale),
                  {output_matmul}),
      perRowPositions(perRowPositions), window(window), rolling(rolling) {
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> AttentionKVCacheObj::inferShape(const TensorVec &ins) {
    IT_ASSERT(ins.size() == 6 || ins.size() == 8, "AttentionKVCache takes 6 inputs, or 8 with an FP8 cache's scales");
    IT_ASSERT(window >= 0, "AttentionKVCache: window " + std::to_string(window) + " is negative (0 = no window)");
    const bool fp8k = ins[0]->getDType() == DataType::Float8E4M3FN, fp8v = ins[1]->getDType() == DataType::Float8E4M3FN;
    // FP8 E4M3 caches (extension): k_scale / v_scale f32 [Hkv] are inputs 6 and 7, present exactly when the caches are FP8
    IT_ASSERT(fp8k == fp8v, "AttentionKVCache: k_cache and v_cache must both be FP8 or neither");
    IT_ASSERT(fp8k == (ins.size() == 8), fp8k ? "AttentionKVCache: an FP8 KV cache needs k_scale and v_scale"
                                              : "AttentionKVCache: k_scale / v_scale go with FP8 caches only");
    if (fp8k) {
        for (int i : {6, 7})
            IT_ASSERT(ins[i]->getDType() == DataType::Float32 && ins[i]->getRank() == 1 && ins[0]->getRank() == 4 &&
                          ins[i]->getDims()[0] == ins[0]->getDims()[1],
                      "AttentionKVCache: k_scale / v_scale must be f32 [Hkv], one scale per KV head");
        for (int i : {2, 3, 4})
            IT_ASSERT(ins[i]->getDType() == DataType::Float16 || ins[i]->getDType() == DataType::BFloat16,
                      "AttentionKVCache: an FP8 KV cache takes f16 / bf16 q, k and v");
        IT_ASSERT(ins[2]->getRank() == 4 && ins[2]->getDims()[2] == 1, "AttentionKVCache: an FP8 KV cache takes one token per step");
    }
    IT_ASSERT(ins[0]->getRank() == 4 && ins[2]->getRank() == 4, "AttentionKVCache expects rank-4 tensors");
    IT_ASSERT(ins[0]->getDims() == ins[1]->getDims(), "k_cache / v_cache shapes differ");
    IT_ASSERT(ins[3]->getDims() == ins[4]->getDims(), "k / v shapes differ");
    IT_ASSERT(ins[3]->getRank() == 4, "AttentionKVCache expects rank-4 tensors");
    // grouped-query attention: caches and k / v carry Hkv heads, q carries Hq = G * Hkv; query head i reads KV head i / G
    const auto &c = ins[0]->getDims(), &q = ins[2]->getDims(), &k = ins[3]->getDims();
    IT_ASSERT(q[0] == c[0] && k[0] == c[0], "AttentionKVCache: batch of q / k / v differs from the caches'");
    IT_ASSERT(q[3] == c[3] && k[3] == c[3], "AttentionKVCache: head dim of q / k / v differs from the caches'");
    IT_ASSERT(k[2] == q[2], "AttentionKVCache: q and k / v lengths differ");
    IT_ASSERT(k[1] == c[1], "AttentionKVCache: k / v head count differs from the caches'");
    IT_ASSERT(c[1] > 0 && q[1] % c[1] == 0, "AttentionKVCache: query heads are not a multiple of the caches' KV heads");
    if (q[2] > 1) {  // a prompt chunk of S tokens at positions p_b .. p_b + S - 1
        IT_ASSERT(q[2] <= c[2], "AttentionKVCache: " + std::to_string(q[2]) + " new tokens do not fit a cache of " +
                                    std::to_string(c[2]) + " rows");
        IT_ASSERT(ins[2]->getDType() != DataType::Float32, "AttentionKVCache: fp32 takes one token per step (S = 1)");
        const int64_t np = (int64_t)ins[5]->size();
        IT_ASSERT(np == (int64_t)q[0] || np == (int64_t)q[0] * q[2],
                  "AttentionKVCache: a prompt chunk takes one position per batch row or one per token");
    }
    if (rolling) {  // a rolling cache (extension): position P in row P mod S_max
        const std::string smax = std::to_string(c[2]), win = std::to_string(window);
        IT_ASSERT(window >= 1, "AttentionKVCache: a rolling cache needs a window >= 1");
        IT_ASSERT(c[2] >= window, "AttentionKVCache: a rolling cache of " + smax + " rows is shorter than the window of " + win);
        IT_ASSERT(c[2] % 64 == 0, "AttentionKVCache: a rolling cache's length " + smax + " is not a multiple of 64");
        IT_ASSERT(c[2] >= (int64_t)window + q[2] - 1,
                  "AttentionKVCache: a chunk of " + std::to_string(q[2]) + " tokens needs a rolling cache of window + " +
                      std::to_string(q[2] - 1) + " = " + std::to_string((int64_t)window + q[2] - 1) + " rows or more, not " +
                      smax + " (split the prompt)");
    }
    return {{ins[2]->getDims()}};
}

SoftmaxObj::SoftmaxObj(GraphObj *graph, Tensor input, Tensor output, int axis)
    : OperatorObj(OpType::Softmax, {input}, {output}), axis(get_real_axis(axis, (int)input->getRank())) {
    IT_ASSERT(checkValid(graph));
}

LayerNormObj::LayerNormObj(GraphObj *graph, Tensor input, Tensor scale, Tensor output, Tensor bias, float eps,
                           int axis, int stash_type)
    : OperatorObj(OpType::LayerNormalization, bias ? TensorVec{input, scale, bias} : TensorVec{input, scale},
                  {output}),
      eps(eps), axis(get_real_axis(axis, (int)input->getRank())), stash_type(stash_type) {
    IT_ASSERT(checkValid(graph));
}

RMSNormObj::RMSNormObj(GraphObj *graph, Tensor input, Tensor weight, Tensor output)
    : OperatorObj(OpType::RMSNorm, {input, weight}, {output}) {
    IT_ASSERT(checkValid(graph));
}

RoPEObj::RoPEObj(GraphObj *graph, Tensor pos, Tensor input, Tensor output, int dimHead, Tensor invFreq)
    : OperatorObj(OpType::RoPE, invFreq ? TensorVec{pos, input, invFreq} : TensorVec{pos, input}, {output}), dimHead(dimHead) {
    IT_ASSERT(dimHead > 0 && dimHead % 2 == 0, "RoPE: dim_head " + std::to_string(dimHead) + " must be positive and even");
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> RoPEObj::inferShape(const TensorVec &ins) {
    IT_ASSERT(ins.size() == 2 || ins.size() == 3, "RoPE takes 2 inputs, or 3 with an inv_freq table");
    if (ins.size() == 3)
        IT_ASSERT(ins[2]->getDType() == DataType::Float32 && ins[2]->getRank() == 1 && ins[2]->getDims()[0] == dimHead / 2,
                  "RoPE: inv_freq must be f32 [dim_head / 2] = [" + std::to_string(dimHead / 2) + "]");
    return {{ins[1]->getDims()}};
}

UnaryObj::UnaryObj(OpType type, GraphObj *graph, Tensor input, Tensor output)
    : OperatorObj(type, {input}, {output}) {
    IT_ASSERT(checkValid(graph));
}

ElementWiseObj::ElementWiseObj(OpType type, GraphObj *graph, Tensor input0, Tensor input1, Tensor output)
    : OperatorObj(type, {input0, input1}, {output}) {
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> ElementWiseObj::inferShape(const TensorVec &ins) {
    return {{infer_broadcast(ins[0]->getDims(), ins[1]->getDims())}};
}
vector<DataType> ElementWiseObj::inferDataType(const TensorVec &ins) const {
    if (type == OpType::Less || type == OpType::Equal || type == OpType::Greater) return {DataType::Bool};
    return {ins[0]->getDType()};
}

TransposeObj::TransposeObj(GraphObj *graph, Tensor input, Tensor output, vector<int> permute)
    : OperatorObj(OpType::Transpose, {input}, {output}) {
    int rank = (int)input->getRank();
    if (permute.empty())
        for (int i = rank - 1; i >= 0; --i) permute.push_back(i);
    IT_ASSERT((int)permute.size() == rank, "Transpose: permutation rank mismatch");
    transposePermute = std::move(permute);
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> TransposeObj::inferShape(const TensorVec &ins) {
    auto &d = ins[0]->getDims();
    Shape out(d.size());
    vector<bool> seen(d.size(), false);
    for (size_t i = 0; i < d.size(); ++i) {
        int p = transposePermute[i];
        IT_ASSERT(p >= 0 && p < (int)d.size() && !seen[p], "Transpose: invalid permutation");
        seen[p] = true;
        out[i] = d[p];
    }
    return {{out}};
}
vector<int> TransposeObj::getOpAttrVector() const {
    vector<int> r{(int)type.underlying()};
    r.insert(r.end(), transposePermute.begin(), transposePermute.end());
    return r;
}

DepthToSpaceObj::DepthToSpaceObj(GraphObj *graph, Tensor input, Tensor output, int blocksize, string mode)
    : OperatorObj(OpType::DepthToSpace, {input}, {output}), blockSize(blocksize), d2sMode(mode == "CRD" ? 1 : 0),
      modeString(mode == "CRD" ? "CRD" : "DCR") {
    IT_ASSERT(blocksize >= 1, "DepthToSpace: blocksize must be positive");
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> DepthToSpaceObj::inferShape(const TensorVec &ins) {
    const auto &d = ins[0]->getDims();
    IT_ASSERT(d.size() == 4, "DepthToSpace expects NCHW");
    const int b = blockSize, c = d[1] / (b * b);
    IT_ASSERT(c * b * b == d[1], "DepthToSpace: channels must be a multiple of blocksize^2");
    // the input viewed as rank 6, and where each of those axes lands (ONNX DepthToSpace: DCR splits the channel axis as
    // (b, b, c), CRD as (c, b, b)); the output interleaves (H, b) and (W, b)
    reshapeDim = d2sMode == 0 ? vector<int>{d[0], b, b, c, d[2], d[3]} : vector<int>{d[0], c, b, b, d[2], d[3]};
    const auto perm = getPermute();
    transposeDim.assign(6, 1);
    for (int i = 0; i < 6; ++i) transposeDim[i] = reshapeDim[perm[i]];
    outDim = {d[0], c, d[2] * b, d[3] * b};
    return {{outDim}};
}

ConcatObj::ConcatObj(GraphObj *graph, TensorVec inputs, Tensor output, int dim_)
    : OperatorObj(OpType::Concat, inputs, {output}) {
    IT_ASSERT(!inputs.empty(), "Concat needs inputs");
    dim = get_real_axis(dim_, (int)inputs[0]->getRank());
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> ConcatObj::inferShape(const TensorVec &ins) {
    Shape out = ins[0]->getDims();
    int total = 0;
    for (auto &t : ins) {
        auto &d = t->getDims();
        IT_ASSERT(d.size() == out.size(), "Concat: rank mismatch");
        for (size_t i = 0; i < d.size(); ++i)
            if ((int)i != dim) IT_ASSERT(d[i] == out[i], "Concat: non-concat dims differ");
        total += d[dim];
    }
    out[dim] = total;
    return {{out}};
}

// src/operators/split.cc:6-58
SplitObj::SplitObj(GraphObj *graph, Tensor input, std::optional<TensorVec> outputs, int dim_, int num_)
    : OperatorObj(OpType::Split, {input}, outputs ? *outputs : TensorVec(num_, nullptr)),
      dim(get_real_axis(dim_, (int)input->getRank())), num(num_) {
    IT_ASSERT(num > 0, "Split: num must be positive");
    int dimSize = input->getDims().at(dim), piece = dimSize / num, last = dimSize - piece * num;
    ratio = vector<int>(num, piece);
    if (last > 0) ratio.back() = piece + last;
    IT_ASSERT(checkValid(graph));
}
SplitObj::SplitObj(GraphObj *graph, Tensor input, std::optional<TensorVec> outputs, int dim_,
                   const vector<int> &ratio_)
    : OperatorObj(OpType::Split, {input}, outputs ? *outputs : TensorVec(ratio_.size(), nullptr)),
      dim(get_real_axis(dim_, (int)input->getRank())), num((int)ratio_.size()), ratio(ratio_) {
    IT_ASSERT(num > 0, "Split: empty ratio");
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> SplitObj::inferShape(const TensorVec &ins) {
    auto d = ins[0]->getDims();
    int total = d.at(dim), sum = std::accumulate(ratio.begin(), ratio.end(), 0);
    IT_ASSERT(sum > 0 && total % sum == 0, "Split: dimension not divisible by the ratio sum");
    int piece = total / sum;
    vector<Shape> ret;
    for (int i = 0; i < num; ++i) {
        d[dim] = piece * ratio[i];
        ret.push_back(d);
    }
    return {ret};
}

GatherObj::GatherObj(GraphObj *graph, Tensor input, Tensor indices, Tensor output, int axis_)
    : OperatorObj(OpType::Gather, {input, indices}, {output}), axis(get_real_axis(axis_, (int)input->getRank())) {
    auto it = indices->getDType();
    IT_ASSERT(it == DataType::Int32 || it == DataType::Int64, "Gather: indices must be int32/int64");
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> GatherObj::inferShape(const TensorVec &ins) {
    auto &d = ins[0]->getDims();
    auto &idx = ins[1]->getDims();
    Shape out(d.begin(), d.begin() + axis);
    out.insert(out.end(), idx.begin(), idx.end());
    out.insert(out.end(), d.begin() + axis + 1, d.end());
    return {{out}};
}

ReshapeObj::ReshapeObj(GraphObj *graph, Tensor input, Tensor output, Shape dims_)
    : OperatorObj(OpType::Reshape, {input}, {output}), dims(std::move(dims_)) {
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> ReshapeObj::inferShape(const TensorVec &ins) {
    Shape out = dims;
    int64_t known = 1;
    int infer = -1;
    for (size_t i = 0; i < out.size(); ++i) {
        if (out[i] == -1) {
            IT_ASSERT(infer < 0, "Reshape: more than one -1");
            infer = (int)i;
        } else {
            if (out[i] == 0 && i < ins[0]->getRank()) out[i] = ins[0]->getDims()[i];
            known *= out[i];
        }
    }
    int64_t total = (int64_t)ins[0]->size();
    if (infer >= 0) {
        IT_ASSERT(known > 0 && total % known == 0, "Reshape: cannot infer -1");
        out[infer] = (int)(total / known);
        known *= out[infer];
    }
    IT_ASSERT(known == total, "Reshape: element count changes");
    return {{out}};
}
FlattenObj::FlattenObj(GraphObj *graph, Tensor input, Tensor output, int axis_)
    : OperatorObj(OpType::Flatten, {input}, {output}) {
    int rank = (int)input->getRank();
    axis = axis_ == rank ? rank : get_real_axis(axis_, rank);
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> FlattenObj::inferShape(const TensorVec &ins) {
    auto &d = ins[0]->getDims();
    int a = 1, b = 1;
    for (int i = 0; i < (int)d.size(); ++i) (i < axis ? a : b) *= d[i];
    return {{{a, b}}};
}
SqueezeObj::SqueezeObj(GraphObj *graph, Tensor input, Tensor output, vector<int> axes_)
    : OperatorObj(OpType::Squeeze, {input}, {output}), axes(std::move(axes_)) {
    for (auto &a : axes) a = get_real_axis(a, (int)input->getRank());
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> SqueezeObj::inferShape(const TensorVec &ins) {
    auto &d = ins[0]->getDims();
    Shape out;
    for (int i = 0; i < (int)d.size(); ++i) {
        bool drop = axes.empty() ? d[i] == 1 : std::find(axes.begin(), axes.end(), i) != axes.end();
        if (drop)
            IT_ASSERT(d[i] == 1, "Squeeze: axis is not of size 1");
        else
            out.push_back(d[i]);
    }
    return {{out}};
}
UnsqueezeObj::UnsqueezeObj(GraphObj *graph, Tensor input, Tensor output, vector<int> axes_)
    : OperatorObj(OpType::Unsqueeze, {input}, {output}), axes(std::move(axes_)) {
    int orank = (int)input->getRank() + (int)axes.size();
    for (auto &a : axes) a = get_real_axis(a, orank);
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> UnsqueezeObj::inferShape(const TensorVec &ins) {
    auto &d = ins[0]->getDims();
    int orank = (int)d.size() + (int)axes.size();
    Shape out(orank, 0);
    for (int a : axes) {
        IT_ASSERT(out[a] == 0, "Unsqueeze: duplicate axis");
        out[a] = 1;
    }
    size_t j = 0;
    for (int i = 0; i < orank; ++i)
        if (out[i] == 0) out[i] = d[j++];
    return {{out}};
}

CastObj::CastObj(GraphObj *graph, Tensor input, Tensor output, DataType to)
    : OperatorObj(OpType::Cast, {input}, {output}), to(to) {
    IT_ASSERT(checkValid(graph));
}

WhereObj::WhereObj(GraphObj *graph, Tensor inputX, Tensor inputY, Tensor condition, Tensor output)
    : OperatorObj(OpType::Where, {inputX, inputY, condition}, {output}) {
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> WhereObj::inferShape(const TensorVec &ins) {
    return {{infer_broadcast(infer_broadcast(ins[0]->getDims(), ins[1]->getDims()), ins[2]->getDims())}};
}

ExpandObj::ExpandObj(GraphObj *graph, Tensor input, Tensor output, Shape dims_)
    : OperatorObj(OpType::Expand, {input}, {output}), dims(std::move(dims_)) {
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> ExpandObj::inferShape(const TensorVec &ins) {
    return {{infer_broadcast(ins[0]->getDims(), dims)}};
}

ReduceBaseObj::ReduceBaseObj(GraphObj *graph, OpType opType, Tensor input, Tensor output,
                             const std::optional<vector<int>> &axes_, bool keepDims)
    : OperatorObj(opType, {input}, {output}), keepDims(keepDims) {
    int rank = (int)input->getRank();
    if (axes_)
        for (int a : *axes_) axes.insert(get_real_axis(a, rank));
    else
        for (int i = 0; i < rank; ++i) axes.insert(i);
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> ReduceBaseObj::inferShape(const TensorVec &ins) {
    auto &d = ins[0]->getDims();
    Shape out;
    for (int i = 0; i < (int)d.size(); ++i) {
        if (!isReduced(i))
            out.push_back(d[i]);
        else if (keepDims)
            out.push_back(1);
    }
    if (out.empty()) out.push_back(1);
    return {{out}};
}

// ONNX Slice incl. negative indices / steps (reference src/operators/slice.cc:9-70)
SliceObj::SliceObj(GraphObj *graph, Tensor input, Tensor output, const vector<int> &starts, const vector<int> &ends,
                   const std::optional<vector<int>> &axes_, const std::optional<vector<int>> &steps_)
    : OperatorObj(OpType::Slice, {input}, {output}) {
    auto &d = input->getDims();
    int rank = (int)d.size();
    IT_ASSERT(starts.size() == ends.size(), "Slice: starts/ends size mismatch");
    axes.resize(rank);
    for (int i = 0; i < rank; ++i) axes[i] = {0, d[i], 1};
    for (size_t i = 0; i < starts.size(); ++i) {
        int a = axes_ ? get_real_axis((*axes_)[i], rank) : (int)i;
        int step = steps_ ? (*steps_)[i] : 1;
        IT_ASSERT(step != 0, "Slice: step 0");
        int len = d[a], s = starts[i], e = ends[i];
        if (s < 0) s += len;
        if (e < 0) e += len;
        if (step > 0) {
            s = std::clamp(s, 0, len);
            e = std::clamp(e, 0, len);
        } else {
            s = std::clamp(s, 0, len - 1);
            e = std::clamp(e, -1, len - 1);
        }
        axes[a] = {s, e, step};
    }
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> SliceObj::inferShape(const TensorVec &) {
    Shape out;
    for (auto &r : axes) {
        int n = r.step > 0 ? (r.end - r.start + r.step - 1) / r.step : (r.start - r.end - r.step - 1) / (-r.step);
        out.push_back(std::max(n, 0));
    }
    return {{out}};
}
vector<int> SliceObj::getStarts() const {
    vector<int> r;
    for (auto &a : axes) r.push_back(a.start);
    return r;
}
vector<int> SliceObj::getSteps() const {
    vector<int> r;
    for (auto &a : axes) r.push_back(a.step);
    return r;
}

PadObj::PadObj(GraphObj *graph, Tensor input, Tensor output, const vector<int> &pads_,
               const std::optional<vector<int>> &axes_)
    : OperatorObj(OpType::Pad, {input}, {output}) {
    int rank = (int)input->getRank();
    pads.assign(rank * 2, 0);
    if (!axes_) {
        IT_ASSERT((int)pads_.size() == rank * 2, "Pad: pads must have 2*rank entries");
        pads = pads_;
    } else {
        size_t n = axes_->size();
        IT_ASSERT(pads_.size() == n * 2, "Pad: pads must have 2*len(axes) entries");
        for (size_t i = 0; i < n; ++i) {
            int a = get_real_axis((*axes_)[i], rank);
            pads[a] = pads_[i];
            pads[a + rank] = pads_[i + n];
        }
    }
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> PadObj::inferShape(const TensorVec &ins) {
    Shape d = ins[0]->getDims();
    int rank = (int)d.size();
    for (int i = 0; i < rank; ++i) {
        IT_ASSERT(pads[i] >= 0 && pads[i + rank] >= 0, "Pad: negative padding");
        d[i] += pads[i] + pads[i + rank];
    }
    return {{d}};
}

PoolingObj::PoolingObj(GraphObj *graph, OpType optype, Tensor input, Tensor output, int kh, int kw, int dh, int dw,
                       int ph, int pw, int sh, int sw, int ceilMode)
    : OperatorObj(optype, {input}, {output}), kh(kh), kw(kw), dh(dh), dw(dw), ph(ph), pw(pw), sh(sh), sw(sw),
      ceilMode(ceilMode) {
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> PoolingObj::inferShape(const TensorVec &ins) {
    Shape d = ins[0]->getDims();
    IT_ASSERT(d.size() == 4, "Pooling expects NCHW");
    auto o = [&](int H, int k, int dil, int p, int s) {
        int num = H + 2 * p - dil * (k - 1) - 1;
        return (ceilMode ? (num + s - 1) / s : num / s) + 1;
    };
    d[2] = o(d[2], kh, dh, ph, sh);
    d[3] = o(d[3], kw, dw, pw, sw);
    return {{d}};
}

BatchNormObj::BatchNormObj(GraphObj *graph, Tensor input, Tensor output, Tensor mean, Tensor var, Tensor scale,
                           Tensor bias, float momentum, float eps, bool trainingMode)
    : OperatorObj(OpType::BatchNormalization, {input, mean, var, scale, bias}, {output}), momentum(momentum),
      eps(eps), trainingMode(trainingMode) {
    IT_ASSERT(!trainingMode, "BatchNormalization: inference only");
    IT_ASSERT(checkValid(graph));
}

AllReduceBaseObj::AllReduceBaseObj(GraphObj *graph, OpType opType, Tensor input, Tensor output)
    : OperatorObj(opType, {input}, {output}) {
    IT_ASSERT(checkValid(graph));
}

AllGatherObj::AllGatherObj(GraphObj *graph, Tensor input, std::optional<TensorVec> outputs, int world_size)
    : OperatorObj(OpType::AllGather, {input}, outputs ? *outputs : TensorVec(world_size, nullptr)),
      world_size(world_size) {
    IT_ASSERT(checkValid(graph));
}
std::optional<vector<Shape>> AllGatherObj::inferShape(const TensorVec &ins) {
    return {vector<Shape>(world_size, ins[0]->getDims())};
}

}  // namespace infini
