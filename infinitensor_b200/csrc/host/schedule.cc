// schedule.cc -- derives the fused execution schedule of a graph (see ExecStep in core.h).
// Pure host logic: pattern matching over the operator list; every fusion keeps the graph-visible results
// bit-identical to the one-kernel-per-operator order the reference runs (src/cuda/cuda_runtime.cc:180-200).
#include <algorithm>
#include <cstdlib>
#include <unordered_map>
#include <unordered_set>

#include "conv_shapes.h"
#include "operators.h"

namespace infini {

static bool fusionEnabled() {
    const char *e = std::getenv("ITB_NO_FUSION");
    return !(e && e[0] == '1');
}
// (bit 9 = NHWC domain for Conv / Pool / Add / Relu chains, on by default)
// (bit 10 = MatMul + bias -> [Gelu] -> [Add] in the wgmma epilogue, on by default)
// (bit 11 = the head split / merge around a prefill-attention chain folded into the attention step, on by default)
// ITB_FUSION_MASK (debug / A-B): bit 0 alias, 1 MatMul groups, 2 MatMul+Add, 3 Silu*Mul, 4 AllReduce+Add+Norm, 5 RoPE->Attention, 6 Conv+BatchNorm[+Add][+Relu], 7 unused; default all
static int fusionMask() {
    const char *e = std::getenv("ITB_FUSION_MASK");
    if (e && e[0]) return std::atoi(e);
    // (bit 8 = prefill attention chains, on by default)
    return 127 | 256 | 512 | 1024 | 2048;
}

static bool isKvCacheOperand(const Tensor &t) {
    for (auto &op : t->getTargets())
        if (op->getOpType() == OpType::AttentionKVCache && (op->getInputs(0) == t || op->getInputs(1) == t)) return true;
    return false;
}
static bool isGraphOutput(const Tensor &t) { return !t->hasTarget() || t->isOutput(); }

// output may share the input's bytes: pure re-interpretation of a contiguous buffer
static bool aliasable(const Operator &op) {
    auto t = op->getOpType();
    bool reshapeLike = t == OpType::Reshape || t == OpType::Flatten || t == OpType::Squeeze || t == OpType::Unsqueeze ||
                       t == OpType::Identity;
    if (t == OpType::Transpose) {
        // a permutation that keeps the relative order of all non-1 dims moves no data
        auto tr = as<TransposeObj>(op);
        auto &d = op->getInputs(0)->getDims();
        int last = -1;
        reshapeLike = true;
        for (int p : tr->getPermute()) {
            if (d[p] == 1) continue;
            if (p < last) reshapeLike = false;
            last = p;
        }
    }
    if (!reshapeLike) return false;
    auto in = op->getInputs(0), out = op->getOutput();
    if (in->getBytes() != out->getBytes()) return false;
    if (isGraphOutput(out) || isKvCacheOperand(in) || isKvCacheOperand(out)) return false;
    return true;
}

static int64_t rowsOf(const Tensor &t) {  // product of all dims but the last
    int64_t r = 1;
    for (size_t i = 0; i + 1 < t->getRank(); ++i) r *= t->getDims()[i];
    return r;
}

static bool groupableMatmul(const Operator &op) {
    auto mm = as<MatmulObj>(op);
    if (!mm || mm->getBias() || mm->getTransA() || mm->getTransB()) return false;
    auto A = mm->getInputs(0), B = mm->getInputs(1);
    auto dt = A->getDType();
    const bool fp8w = mm->getWScale() != nullptr;  // FP8 weight + per-column scale: grouped only with its own kind (checked by the caller)
    if (!(dt == DataType::Float16 || dt == DataType::BFloat16) || (!fp8w && B->getDType() != dt)) return false;
    if (B->getRank() != 2 || !B->isWeight()) return false;
    if (rowsOf(A) > 64) return false;  // decode regime: the grouped kernel is the skinny GEMM
    return true;
}

// Multi-token attention as the frontend lowers it (no fused op exists in the reference for q-len > 1):
//   kt = Transpose(k, swap of the last two axes); s = MatMul(q, kt); [s = Div | Mul(s, scalar)]; [s = Add(s, mask)];
//   p = Softmax(s, axis -1); out = MatMul(p, v)         q [B,H,Sq,D], k / v [B,H,Skv,D], D in {64, 128}, f16 / bf16
// every link single-consumer.  Returns the chain {transpose, mm1, [scale], [add], softmax} for `mm2`, or empty.
static OpVec matchPrefillChain(const Operator &mm2op) {
    auto mm2 = as<MatmulObj>(mm2op);
    if (!mm2 || mm2->getBias() || mm2->getTransA() || mm2->getTransB()) return {};
    Tensor p = mm2->getInputs(0), v = mm2->getInputs(1);
    auto half = [](const Tensor &t) { return t->getDType() == DataType::Float16 || t->getDType() == DataType::BFloat16; };
    if (!half(p) || v->getDType() != p->getDType() || p->getRank() != 4 || v->getRank() != 4) return {};
    auto sole = [](const Tensor &t) { return !t->isOutput() && t->getTargets().size() == 1; };
    auto sm = p->getSource();
    if (!sm || sm->getOpType() != OpType::Softmax || !sole(p) || as<SoftmaxObj>(sm)->getAxis() != 3) return {};
    OpVec mid;
    Tensor s = sm->getInputs(0);
    auto src = s->getSource();
    if (src && src->getOpType() == OpType::Add && sole(s)) {
        // one operand continues the chain, the other is the mask (anything produced outside the chain, broadcastable)
        Tensor a0 = src->getInputs(0), a1 = src->getInputs(1);
        auto chainish = [](const Tensor &t) {
            auto o = t->getSource();
            return o && (o->getOpType() == OpType::MatMul || o->getOpType() == OpType::Div || o->getOpType() == OpType::Mul);
        };
        Tensor cont = chainish(a0) ? a0 : chainish(a1) ? a1 : nullptr;
        if (!cont || cont->getDims() != s->getDims()) return {};
        Tensor other = cont == a0 ? a1 : a0;
        if (other->getDType() != s->getDType() || other->getRank() > 4) return {};
        mid.insert(mid.begin(), src);
        s = cont;
        src = s->getSource();
    }
    if (src && (src->getOpType() == OpType::Div || src->getOpType() == OpType::Mul) && sole(s)) {
        Tensor a0 = src->getInputs(0), a1 = src->getInputs(1);
        const bool isDiv = src->getOpType() == OpType::Div;
        Tensor cont = (a1->size() == 1 && !a1->getSource()) ? a0 : (!isDiv && a0->size() == 1 && !a0->getSource()) ? a1 : nullptr;
        if (!cont || cont->getDims() != s->getDims()) return {};
        Tensor scalar = cont == a0 ? a1 : a0;
        if (scalar->getDType() != s->getDType()) return {};
        mid.insert(mid.begin(), src);
        s = cont;
        src = s->getSource();
    }
    auto mm1 = src ? as<MatmulObj>(src) : nullptr;
    if (!mm1 || !sole(s) || mm1->getBias() || mm1->getTransA() || mm1->getTransB()) return {};
    Tensor q = mm1->getInputs(0), kt = mm1->getInputs(1);
    auto tr = kt->getSource() ? as<TransposeObj>(kt->getSource()) : nullptr;
    if (!tr || !sole(kt) || tr->getPermute() != vector<int>{0, 1, 3, 2}) return {};
    Tensor k = tr->getInputs(0);
    if (q->getRank() != 4 || k->getRank() != 4 || q->getDType() != p->getDType() || k->getDType() != p->getDType()) return {};
    auto &qd = q->getDims();
    auto &kd = k->getDims();
    auto &vd = v->getDims();
    const int D = qd[3];
    if ((D != 64 && D != 128) || kd[3] != D || vd[3] != D || kd[0] != qd[0] || kd[1] != qd[1] || vd[0] != qd[0] || vd[1] != qd[1] ||
        vd[2] != kd[2])
        return {};
    OpVec chain = {kt->getSource(), src};
    chain.insert(chain.end(), mid.begin(), mid.end());
    chain.push_back(sm);
    return chain;
}

// The frontend's head split / merge around a prefill-attention chain (GPT-2):
//   qkv [B, S, 3 H D] -> Split(axis 2, 3) -> 3 x { Reshape [B, S, H, D] -> Transpose [0,2,1,3] } -> chain -> Transpose [0,2,1,3] -> Reshape [B, S, H D]
// When every link has a single consumer the whole neighbourhood runs as ONE PrefillAttention step: q / k / v become strided views of
// the projection output and the result is written in its final layout (it_b200_attention_prefill_strided).  Returns the operators
// in execution order -- {Split, Rq, Tq, Rk, Tk, Rv, Tv, <chain>, mm2, Tout, Rout} -- or {} when the pattern is not there.
static OpVec extendPrefillChain(const OpVec &chain, const Operator &mm2op) {
    auto sole = [](const Tensor &t) { return !t->isOutput() && t->getTargets().size() == 1; };
    auto mm1 = chain[1];
    Tensor q = mm1->getInputs(0), k = chain[0]->getInputs(0), v = mm2op->getInputs(1);
    const vector<int> perm = {0, 2, 1, 3};
    Operator split;
    OpVec pre;
    int part = 0;
    for (auto &t : {q, k, v}) {
        auto tr = t->getSource() ? as<TransposeObj>(t->getSource()) : nullptr;
        if (!tr || !sole(t) || tr->getPermute() != perm) return {};
        Tensor r = tr->getInputs(0);
        auto rs = r->getSource();
        if (!rs || rs->getOpType() != OpType::Reshape || !sole(r) || r->getRank() != 4) return {};
        Tensor piece = rs->getInputs(0);
        auto sp = piece->getSource() ? as<SplitObj>(piece->getSource()) : nullptr;
        if (!sp || !sole(piece) || piece->getRank() != 3 || sp->getDim() != 2 || sp->numOutputs() != 3) return {};
        if (split && sp != split) return {};
        split = sp;
        if (sp->getOutputs()[part] != piece) return {};  // q, k, v = parts 0, 1, 2 in this order
        auto &pd = piece->getDims();
        auto &rd = r->getDims();
        if (rd[0] != pd[0] || rd[1] != pd[1] || rd[2] * rd[3] != pd[2]) return {};
        pre.push_back(rs);
        pre.push_back(tr);
        ++part;
    }
    auto &d0 = split->getOutputs()[0]->getDims();
    for (auto &o : split->getOutputs())
        if (o->getDims() != d0) return {};
    Tensor o = mm2op->getOutput();
    if (!sole(o)) return {};
    auto tout = as<TransposeObj>(o->getTargets()[0]);
    if (!tout || tout->getPermute() != perm || !sole(tout->getOutput())) return {};
    auto rout = tout->getOutput()->getTargets()[0];
    if (rout->getOpType() != OpType::Reshape) return {};
    auto &od = rout->getOutput()->getDims();
    auto &qd = q->getDims();
    if (od.size() != 3 || od[0] != qd[0] || od[1] != qd[2] || od[2] != qd[1] * qd[3]) return {};
    OpVec all = {split};
    all.insert(all.end(), pre.begin(), pre.end());
    all.insert(all.end(), chain.begin(), chain.end());
    all.push_back(mm2op);
    all.push_back(tout);
    all.push_back(rout);
    return all;
}

// ---------------------------------------------------------------- NHWC domain
// ResNet-style chains run fastest with channel-innermost activations: the implicit-GEMM conv (kernels/conv_nhwc.cu) reads them
// through the TMA unit's im2col mode and no im2col matrix is ever written.  A tensor is stored NHWC only when EVERY step touching
// it can work in that layout; the decision is a fixpoint over the schedule:
//   Conv / Conv+BN[+Add][+Relu] : NHWC input needs the implicit-GEMM kernel's shape limits (it_b200_conv2d_nhwc_supported); its
//                                 output (and residual, which must agree with the output) may be either layout.  With an NCHW
//                                 input (the 3-channel stem) the im2col GEMM can still WRITE NHWC (it_b200_conv2d_nchw_to_nhwc_supported)
//   MaxPool / AvgPool           : input and output agree (C % 8 == 0 for the NHWC kernel)
//   Relu / Add of equal shapes  : flat elementwise, operands and result agree
//   anything else, graph inputs / outputs / weights: NCHW
// A [N, C, 1, 1] tensor is the same bytes either way and never constrains anything.
namespace {
struct LayoutPass {
    enum Cls { Other, ConvStep, PoolStep, EltStep };
    std::unordered_set<TensorObj *> nhwc;

    static bool free4(const Tensor &t) {
        auto &d = t->getDims();
        return d.size() == 4 && d[2] * d[3] == 1;
    }
    static bool candidate(const Tensor &t) {
        auto &d = t->getDims();
        if (d.size() != 4 || free4(t)) return false;
        auto dt = t->getDType();
        if (!(dt == DataType::Float16 || dt == DataType::BFloat16)) return false;
        return !t->isWeight() && !t->isInput() && !t->isOutput() && t->getSource() && !t->getTargets().empty();
    }
    static Cls classify(const ExecStep &st) {
        const auto &op = st.ops.back();
        if (st.kind == ExecStep::ConvBnAct) return ConvStep;
        if (st.kind != ExecStep::Single) return Other;
        auto ty = op->getOpType();
        if (ty == OpType::Conv) return ConvStep;
        if (ty == OpType::MaxPool || ty == OpType::AveragePool) {
            auto &d = op->getInputs(0)->getDims();
            return d.size() == 4 && d[1] % 8 == 0 ? PoolStep : Other;
        }
        if (ty == OpType::Relu) return EltStep;
        if (ty == OpType::Add) {
            auto &a = op->getInputs(0)->getDims(), &b = op->getInputs(1)->getDims();
            return a == b && a == op->getOutput()->getDims() ? EltStep : Other;
        }
        return Other;
    }
    static Tensor convResidual(const ExecStep &st) {
        for (size_t i = 2; i < st.ops.size(); ++i)
            if (st.ops[i]->getOpType() == OpType::Add) {
                Tensor prev = st.ops[i - 1]->getOutput();
                return st.ops[i]->getInputs(0) == prev ? st.ops[i]->getInputs(1) : st.ops[i]->getInputs(0);
            }
        return nullptr;
    }
    bool is(const Tensor &t) const { return t && nhwc.count(t.get()) > 0; }
    bool drop(const Tensor &t) { return t && nhwc.erase(t.get()) > 0; }

    void run(vector<ExecStep> &schedule) {
        // tensors written / read INSIDE a fused step never exist in memory; everything else a step touches is "external"
        for (auto &st : schedule)
            for (auto &op : st.ops) {
                for (auto &t : op->getInputs())
                    if (candidate(t)) nhwc.insert(t.get());
                for (auto &t : op->getOutputs())
                    if (candidate(t)) nhwc.insert(t.get());
            }
        bool changed = true;
        while (changed) {
            changed = false;
            for (auto &st : schedule) {
                Cls c = classify(st);
                if (c == ConvStep) {
                    auto conv = as<ConvObj>(st.ops[0]);
                    Tensor x = conv->getInputs(0), y = st.ops.back()->getOutput(), res = convResidual(st);
                    auto [n, ci, h, w, f, r, s] = conv->getNCHWFRS();
                    auto [ph, pw, sh, sw, dh, dw] = conv->getPadStrideDilation();
                    const int g = conv->getNumGroups(), dt = x->getDType().getIndex();
                    // operands of the chain other than x / residual (weights, statistics) are never candidates
                    if (is(x) && !itb::conv_nhwc_ok(dt, ci, f, r, s, ph, pw, sh, sw, dh, dw, g)) changed |= drop(x);
                    if (is(y) && !is(x)) {
                        // an NCHW input can still enter the domain: the stem kernel (<= 4 channels, no residual) or the
                        // folded im2col GEMM scattering its result channel-innermost
                        const bool stem = !res && itb::conv_stem_ok(dt, ci, f, r, s, ph, pw, sh, sw, dh, dw, g);
                        if (!stem && !itb::conv_nchw_to_nhwc_ok(dt, n, ci, h, w, f, r, s, ph, pw, sh, sw, dh, dw, g)) changed |= drop(y);
                    }
                    if (res && !free4(res) && is(res) != is(y)) {
                        changed |= drop(res);
                        changed |= drop(y);
                    }
                    // everything else the chain reads (filters, statistics) is consumed in the reference's own order
                    for (auto &m : st.ops)
                        for (auto &t : m->getInputs())
                            if (t != x && t != res) changed |= drop(t);
                } else if (c == PoolStep || c == EltStep) {
                    const auto &op = st.ops.back();
                    bool all = true;
                    auto visit = [&](const Tensor &t) {
                        if (t->getDims().size() == 4 && !free4(t) && !is(t)) all = false;
                    };
                    for (auto &t : op->getInputs()) visit(t);
                    visit(op->getOutput());
                    if (!all) {
                        for (auto &t : op->getInputs()) changed |= drop(t);
                        changed |= drop(op->getOutput());
                    }
                } else {
                    for (auto &op : st.ops) {
                        for (auto &t : op->getInputs()) changed |= drop(t);
                        for (auto &t : op->getOutputs()) changed |= drop(t);
                    }
                }
            }
        }
        for (auto &st : schedule) {
            Cls c = classify(st);
            if (c == Other) continue;
            const auto &last = st.ops.back();
            const Tensor x = st.ops[0]->getInputs(0), y = last->getOutput();
            bool in = is(x), out = is(y);
            if (c != ConvStep) {
                // (a pooled [N, C, 1, 1] result is layout-free: the NHWC kernel writes the same bytes)
                for (auto &t : last->getInputs()) in = in || is(t);
                out = out || (in && free4(y));
                in = in || (out && free4(x));
                if (in != out) in = out = false;  // cannot happen after the fixpoint; stay on the NCHW kernels
            }
            st.layout = (in ? 1 : 0) | (out ? 2 : 0);
        }
    }
};
}  // namespace

const vector<ExecStep> &GraphObj::getSchedule() {
    if (scheduleEpoch == getTopologyEpoch() && !schedule.empty()) return schedule;
    IT_ASSERT(topo_sort(), "graph has a cycle");
    schedule.clear();
    const bool fuse = fusionEnabled();
    const int mask = fusionMask();
    std::unordered_map<OperatorObj *, int> pos;
    for (size_t i = 0; i < ops.size(); ++i) pos[ops[i].get()] = (int)i;
    std::unordered_set<OperatorObj *> consumed;               // executed as part of an earlier (horizontal) step
    std::unordered_map<OperatorObj *, OpVec> deferredInto;  // consumer -> producer(s) executed with it
    std::unordered_set<OperatorObj *> deferred;

    // prefill attention chains first: their members must not be claimed by the per-operator patterns below
    if (fuse && (mask & 256))
        for (auto &op : ops) {
            if (op->getOpType() != OpType::MatMul) continue;
            OpVec chain = matchPrefillChain(op);
            if (chain.empty()) continue;
            bool clash = deferredInto.count(op.get()) > 0;
            for (auto &m : chain) clash = clash || deferred.count(m.get()) || deferredInto.count(m.get());
            if (clash) continue;
            if (mask & 2048) {
                // with the head split / merge around it: everything is parked behind the final Reshape
                OpVec all = extendPrefillChain(chain, op);
                bool ok = !all.empty();
                for (auto &m : all) ok = ok && !deferred.count(m.get()) && !deferredInto.count(m.get());
                if (ok) {
                    auto last = all.back();
                    all.pop_back();
                    for (auto &m : all) deferred.insert(m.get());
                    deferredInto[last.get()] = all;
                    continue;
                }
            }
            for (auto &m : chain) deferred.insert(m.get());
            deferredInto[op.get()] = chain;
        }

    for (size_t i = 0; i < ops.size(); ++i) {
        const Operator &op = ops[i];
        if (consumed.count(op.get()) || deferred.count(op.get())) continue;
        ExecStep st;
        st.ops = {op};
        auto it = deferredInto.find(op.get());
        if (it != deferredInto.end()) {
            const OpVec &prod = it->second;
            auto pt = prod[0]->getOpType();
            if (pt == OpType::Transpose || pt == OpType::Split) {  // (Split first: the chain with its head split / merge)
                st.kind = ExecStep::PrefillAttention;
                st.ops = prod;
                st.ops.push_back(op);
                schedule.push_back(std::move(st));
                continue;
            }
            if (pt == OpType::RoPE) {
                // both RoPE(q) and RoPE(k) must have been folded; a lone one simply runs here, just before its consumer
                Operator rq, rk;
                for (auto &r : prod) {
                    Tensor t = r->getOutput();
                    while (t->getTargets().size() == 1 && t->getTargets()[0] != op) t = t->getTargets()[0]->getOutput();
                    if (t == op->getInputs(2)) rq = r;
                    if (t == op->getInputs(3)) rk = r;
                }
                // angles from one rule: the same inv_freq table tensor, or the base-10000 rule for both
                if (rq && rk && rq != rk && as<RoPEObj>(rq)->getInvFreq() == as<RoPEObj>(rk)->getInvFreq()) {
                    st.kind = ExecStep::AttentionRope;
                    st.ops = {rq, rk, op};
                } else {
                    for (auto &r : prod) {
                        ExecStep single;
                        single.ops = {r};
                        schedule.push_back(std::move(single));
                    }
                }
                schedule.push_back(std::move(st));
                continue;
            }
            if (pt == OpType::Conv) {
                st.kind = ExecStep::ConvBnAct;
                st.ops = prod;
                st.ops.push_back(op);
                schedule.push_back(std::move(st));
                continue;
            }
            st.kind = pt == OpType::MatMul || pt == OpType::MatMulNBits ? ExecStep::MatMulAdd : pt == OpType::Silu ? ExecStep::SiluMul : ExecStep::AllReduceAddNorm;
            st.ops = prod;  // MatMulAdd: {MatMul, [activation], Add | activation}; the others: one producer
            st.ops.push_back(op);
            if (st.kind == ExecStep::AllReduceAddNorm) {
                // pull in the RMSNorm that normalises the new residual stream (executed early, with the Add)
                for (auto &t : op->getOutput()->getTargets())
                    if (t->getOpType() == OpType::RMSNorm && t->getInputs(0) == op->getOutput() && !consumed.count(t.get()) &&
                        !deferred.count(t.get()) && t->getInputs(1)->isWeight()) {
                        st.ops.push_back(t);
                        consumed.insert(t.get());
                        break;
                    }
            }
            schedule.push_back(std::move(st));
            continue;
        }
        if (!fuse) {
            schedule.push_back(std::move(st));
            continue;
        }
        const auto type = op->getOpType();
        if ((mask & 1) && aliasable(op)) {
            st.kind = ExecStep::Alias;
        } else if (type == OpType::MatMul) {
            // (1) horizontal: later MatMuls reading the same activation tensor
            if ((mask & 2) && groupableMatmul(op)) {
                auto A = op->getInputs(0);
                int k = as<MatmulObj>(op)->getK();
                for (auto &cand : A->getTargets()) {
                    if (st.ops.size() >= 4) break;
                    if (cand == op || consumed.count(cand.get()) || deferred.count(cand.get())) continue;
                    if (cand->getOpType() != OpType::MatMul || cand->getInputs(0) != A) continue;
                    if (pos[cand.get()] < (int)i || !groupableMatmul(cand) || as<MatmulObj>(cand)->getK() != k) continue;
                    if ((as<MatmulObj>(cand)->getWScale() != nullptr) != (as<MatmulObj>(op)->getWScale() != nullptr)) continue;
                    st.ops.push_back(cand);
                }
                if (st.ops.size() > 1) {
                    st.kind = ExecStep::MatMulGroup;
                    std::sort(st.ops.begin(), st.ops.end(),
                              [&](const Operator &a, const Operator &b) { return pos[a.get()] < pos[b.get()]; });
                    for (size_t j = 1; j < st.ops.size(); ++j) consumed.insert(st.ops[j].get());
                }
            }
            // (2) vertical: MatMul -> Add(residual of identical shape), executed at the Add's position
            if (st.kind == ExecStep::Single && (mask & 4)) {
                auto mm = as<MatmulObj>(op);
                auto out = op->getOutput();
                auto targets = out->getTargets();
                // a biased Linear layer (Gemm: GPT-2's c_attn / c_proj / c_fc) or an activation between MatMul and Add needs the
                // wgmma epilogue (it_b200_matmul_fused): f16 / bf16, more than 64 rows, plain [.., K] x [K, N]
                auto fusedShape = [&]() {
                    auto A = op->getInputs(0), Bw = op->getInputs(1);
                    auto dt = out->getDType();
                    if (!(dt == DataType::Float16 || dt == DataType::BFloat16) || mm->getTransA() || mm->getWScale()) return false;
                    if (Bw->getRank() != 2 && A->getRank() != Bw->getRank()) return false;
                    int64_t rows = 1;
                    for (size_t i = 0; i + 1 < A->getRank(); ++i) rows *= A->getDims()[i];
                    return rows > 64 && mm->getK() % 8 == 0 && mm->getN() % 8 == 0 && mm->getK() >= 64 && mm->getN() >= 64;
                };
                auto freeOp = [&](const Operator &o) {
                    return !deferredInto.count(o.get()) && !deferred.count(o.get()) && !consumed.count(o.get());
                };
                OpVec chain = {op};
                Tensor t = out;
                bool ok = out->getDType().isFloat() && targets.size() == 1 && !out->isOutput() && freeOp(targets[0]);
                if (ok && targets[0]->getOpType() == OpType::Gelu && (mask & 1024) && fusedShape() &&
                    targets[0]->getOutput()->getDims() == out->getDims()) {
                    chain.push_back(targets[0]);  // MatMul -> Gelu
                    t = targets[0]->getOutput();
                    auto tt = t->getTargets();
                    ok = tt.size() == 1 && !t->isOutput() && freeOp(tt[0]);
                    targets = tt;
                }
                bool withAdd = false;
                if (ok && targets[0]->getOpType() == OpType::Add && (!mm->getBias() || ((mask & 1024) && fusedShape())) &&
                    (chain.size() == 1 || fusedShape())) {
                    auto add = targets[0];
                    auto other = add->getInputs(0) == t ? add->getInputs(1) : add->getInputs(0);
                    if (other != t && other->getDims() == t->getDims() && other->getDType() == t->getDType() &&
                        add->getOutput()->getDims() == t->getDims()) {
                        chain.push_back(add);
                        withAdd = true;
                    }
                }
                if (chain.size() > 1) {
                    (void)withAdd;
                    auto last = chain.back();
                    chain.pop_back();
                    deferredInto[last.get()] = chain;
                    for (auto &m : chain) deferred.insert(m.get());
                    continue;
                }
            }
        } else if (type == OpType::MatMulNBits) {
            // the 4-bit MatMul takes the same two fusions as the 16-bit one: (1) later MatMulNBits reading the same activation with
            // the same K, block size and zero-point presence, in the decode regime, run as one grouped launch; (2) MatMulNBits ->
            // Add(residual of identical shape) runs at the Add's position with the residual added after the product is rounded
            auto nb = as<MatMulNBitsObj>(op);
            auto A = op->getInputs(0);
            auto like = [&](const Operator &c) {
                auto o = as<MatMulNBitsObj>(c);
                return o && c->getInputs(0) == A && o->getK() == nb->getK() && o->getBlockSize() == nb->getBlockSize() &&
                       (o->getZeroPoints() != nullptr) == (nb->getZeroPoints() != nullptr);
            };
            if ((mask & 2) && rowsOf(A) <= 64) {
                for (auto &cand : A->getTargets()) {
                    if (st.ops.size() >= 4) break;
                    if (cand == op || consumed.count(cand.get()) || deferred.count(cand.get()) || pos[cand.get()] < (int)i) continue;
                    if (like(cand)) st.ops.push_back(cand);
                }
                if (st.ops.size() > 1) {
                    st.kind = ExecStep::MatMulGroup;
                    std::sort(st.ops.begin(), st.ops.end(),
                              [&](const Operator &a, const Operator &b) { return pos[a.get()] < pos[b.get()]; });
                    for (size_t j = 1; j < st.ops.size(); ++j) consumed.insert(st.ops[j].get());
                }
            }
            auto out = op->getOutput();
            auto targets = out->getTargets();
            if (st.kind == ExecStep::Single && (mask & 4) && targets.size() == 1 && !out->isOutput() &&
                targets[0]->getOpType() == OpType::Add && !deferredInto.count(targets[0].get()) && !deferred.count(targets[0].get()) &&
                !consumed.count(targets[0].get())) {
                auto add = targets[0];
                auto other = add->getInputs(0) == out ? add->getInputs(1) : add->getInputs(0);
                if (other != out && other->getDims() == out->getDims() && other->getDType() == out->getDType() &&
                    add->getOutput()->getDims() == out->getDims()) {
                    deferredInto[add.get()] = {op};
                    deferred.insert(op.get());
                    continue;
                }
            }
        } else if (type == OpType::RoPE && (mask & 32)) {
            // RoPE -> (alias-only chain) -> AttentionKVCache q / k operand, S = 1, heads of the RoPE's width D in {64, 128}:
            // fold into the attention kernel.  A RoPE whose width is not the cache's head width runs unfused.
            const int dh = as<RoPEObj>(op)->getDimHead();
            Tensor t = op->getOutput();
            bool chain = !t->isOutput();
            while (chain && t->getTargets().size() == 1 && (mask & 1) && aliasable(t->getTargets()[0])) t = t->getTargets()[0]->getOutput();
            auto &xd = op->getInputs(1)->getDims();
            if (chain && t->getTargets().size() == 1 && t->getTargets()[0]->getOpType() == OpType::AttentionKVCache &&
                (dh == 64 || dh == 128) && xd.size() == 3 && xd[1] == 1 && xd[2] % dh == 0 && op->getInputs(1)->getDType().isFloat()) {
                auto att = t->getTargets()[0];
                // the operand this RoPE feeds: q carries Hq heads, k the caches' Hkv (fewer under grouped-query attention)
                auto &qd = (att->getInputs(2) == t ? att->getInputs(2) : att->getInputs(3))->getDims();
                if ((att->getInputs(2) == t || att->getInputs(3) == t) && qd[2] == 1 && qd[3] == dh && qd[0] == xd[0] &&
                    qd[1] * dh == xd[2]) {
                    deferredInto[att.get()].push_back(op);
                    deferred.insert(op.get());
                    continue;
                }
            }
        } else if (type == OpType::AllReduceSum && (mask & 16)) {
            auto out = op->getOutput();
            auto targets = out->getTargets();
            if (out->getDType().isFloat() && targets.size() == 1 && !out->isOutput() && targets[0]->getOpType() == OpType::Add &&
                !deferredInto.count(targets[0].get()) && !deferred.count(targets[0].get()) && !consumed.count(targets[0].get())) {
                auto add = targets[0];
                auto other = add->getInputs(0) == out ? add->getInputs(1) : add->getInputs(0);
                if (other != out && other->getDims() == out->getDims() && other->getDType() == out->getDType() &&
                    add->getOutput()->getDims() == out->getDims()) {
                    deferredInto[add.get()] = {op};
                    deferred.insert(op.get());
                    continue;
                }
            }
        } else if (type == OpType::Conv && (mask & 64)) {
            // Conv -> BatchNorm -> [Add(x, same shape)] -> [Relu], every link single-consumer: the chain runs as ONE step at
            // the position of its last operator (the Add's other operand is then already computed)
            OpVec chain = {op};
            Tensor t = op->getOutput();
            auto sole = [&](const Tensor &x) -> Operator {
                if (x->isOutput() || x->getTargets().size() != 1) return nullptr;
                auto c = x->getTargets()[0];
                if (consumed.count(c.get()) || deferred.count(c.get()) || deferredInto.count(c.get())) return nullptr;
                return c;
            };
            Operator nx = sole(t);
            if (t->getDType().isFloat() && nx && nx->getOpType() == OpType::BatchNormalization && nx->getInputs(0) == t) {
                bool statsOk = true;
                for (int k = 1; k <= 4; ++k) statsOk = statsOk && nx->getInputs(k)->getDType() == DataType::Float32;
                if (statsOk) {
                    chain.push_back(nx);
                    t = nx->getOutput();
                    nx = sole(t);
                    if (nx && nx->getOpType() == OpType::Add) {
                        auto other = nx->getInputs(0) == t ? nx->getInputs(1) : nx->getInputs(0);
                        if (other != t && other->getDims() == t->getDims() && other->getDType() == t->getDType() &&
                            nx->getOutput()->getDims() == t->getDims()) {
                            chain.push_back(nx);
                            t = nx->getOutput();
                            nx = sole(t);
                        }
                    }
                    if (nx && nx->getOpType() == OpType::Relu && nx->getInputs(0) == t) chain.push_back(nx);
                    auto last = chain.back();
                    chain.pop_back();
                    deferredInto[last.get()] = chain;
                    for (auto &m : chain) deferred.insert(m.get());
                    continue;
                }
            }
        } else if (type == OpType::Silu && (mask & 8)) {
            auto out = op->getOutput();
            auto targets = out->getTargets();
            if (targets.size() == 1 && !out->isOutput() && targets[0]->getOpType() == OpType::Mul &&
                !deferredInto.count(targets[0].get()) && !deferred.count(targets[0].get()) && !consumed.count(targets[0].get())) {
                auto mul = targets[0];
                auto other = mul->getInputs(0) == out ? mul->getInputs(1) : mul->getInputs(0);
                if (other != out && other->getDims() == out->getDims() && other->getDType() == out->getDType() &&
                    mul->getOutput()->getDims() == out->getDims()) {
                    deferredInto[mul.get()] = {op};
                    deferred.insert(op.get());
                    continue;
                }
            }
        }
        schedule.push_back(std::move(st));
    }
    if (fuse && (mask & 512)) LayoutPass().run(schedule);
    // every operator is executed by exactly one step (a producer parked behind a consumer that never runs would be a
    // silently skipped op)
    {
        std::unordered_map<OperatorObj *, int> seen;
        for (auto &stp : schedule)
            for (auto &m : stp.ops) ++seen[m.get()];
        for (auto &o : ops) IT_ASSERT(seen[o.get()] == 1, "schedule: operator " + o->toString() + " is not covered by exactly one step");
    }
    scheduleEpoch = topologyEpoch;
    return schedule;
}

}  // namespace infini
