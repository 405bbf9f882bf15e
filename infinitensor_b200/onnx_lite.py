"""ONNX ingestion without the `onnx` package (SURVEY.md 8(f-1)).

The reference drives its backend through `OnnxStub(model, runtime)` (pyinfinitensor/src/pyinfinitensor/onnx.py:41-1136):
one `handler.<op>(...)` call per ONNX node.  That module needs `onnx` + `onnxsim`, which this image does not have, so this
file carries the two pieces the path needs from them and nothing else:

  * a protobuf WIRE reader / writer for the handful of ONNX messages involved (ModelProto, GraphProto, NodeProto,
    AttributeProto, TensorProto, ValueInfoProto; field numbers from onnx.proto3, IR version 8) -- `load_model`,
    `save_model`;
  * `OnnxStub`: the node -> handler-call lowering for every operator this backend has a kernel for, with the
    reference frontend's conventions (quirk ledger q12): dynamic dims become 1 (onnx.py:1625-1626), Gemm needs
    alpha = beta = 1 (:298-300), Conv bias becomes Reshape + Add (:159-190), asymmetric Conv pads become an explicit
    Pad (:150-155), GlobalAveragePool becomes AveragePool with k = (H, W) (:489-503), Dropout becomes Identity
    (:898-910), ReduceSum with a `communicator` attribute becomes AllReduceSum (:917-923), Constant nodes and
    initializers become weight tensors.

`OnnxStub` takes any object with the GraphHandler surface (backend.GraphHandler in the product; the CPU tests hand it the
oracle's handler).  onnxsim is replaced by the one thing the reference needs it for: COMPILE-TIME CONSTANT FOLDING of the
shape arithmetic exporters emit (Shape -> Gather -> Unsqueeze -> Concat -> Reshape, ConstantOfShape / Range / Equal / Where
mask builders, Cast / Slice / Mul on those...).  All shapes are static here, so `Shape` of any tensor is a constant and
every node whose inputs are constants is evaluated with numpy at load time (`_FOLD`); constants become device weights only
when a lowered operator actually consumes them.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import numpy as np

# ONNX TensorProto.DataType codes used by the backend (include/core/data_type.h:6-23 has the same numbering)
F32, U8, I8, I16, I32, I64, BOOL, F16, F64, U32, BF16, FP8 = 1, 2, 3, 5, 6, 7, 9, 10, 11, 12, 16, 17
_NP = {F32: np.float32, U8: np.uint8, I8: np.int8, I16: np.int16, I32: np.int32, I64: np.int64, BOOL: np.bool_,
       F16: np.float16, F64: np.float64, U32: np.uint32, BF16: np.uint16, FP8: np.uint8}  # FP8: E4M3 "FN" codes


# ------------------------------------------------------------------------------------------------ wire format
def _varint(buf, i):
    r = s = 0
    while True:
        b = buf[i]
        i += 1
        r |= (b & 0x7F) << s
        if b < 0x80:
            return r, i
        s += 7


def _fields(buf):
    """(field number, wire type, value) triples of one message; length-delimited values are memoryviews."""
    buf = memoryview(buf)
    i, n = 0, len(buf)
    while i < n:
        key, i = _varint(buf, i)
        no, wt = key >> 3, key & 7
        if wt == 0:
            v, i = _varint(buf, i)
        elif wt == 1:
            v, i = bytes(buf[i:i + 8]), i + 8
        elif wt == 2:
            ln, i = _varint(buf, i)
            v, i = buf[i:i + ln], i + ln
        elif wt == 5:
            v, i = bytes(buf[i:i + 4]), i + 4
        else:
            raise ValueError(f"protobuf wire type {wt} not supported")
        yield no, wt, v


def _sint64(v):  # int64 fields carry negatives as 64-bit two's complement varints
    return v - (1 << 64) if v >= (1 << 63) else v


def _packed_ints(wt, v):
    if wt == 0:
        return [_sint64(v)]
    out, i = [], 0
    while i < len(v):
        x, i = _varint(v, i)
        out.append(_sint64(x))
    return out


def _packed_f32(wt, v):
    return list(struct.unpack("<f", v)) if wt == 5 else list(np.frombuffer(v, dtype="<f4"))


def _enc_varint(x):
    x &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = x & 0x7F
        x >>= 7
        out.append(b | (0x80 if x else 0))
        if not x:
            return bytes(out)


def _key(no, wt):
    return _enc_varint((no << 3) | wt)


def _ld(no, payload: bytes):
    return _key(no, 2) + _enc_varint(len(payload)) + payload


# ------------------------------------------------------------------------------------------------ messages
@dataclass
class TensorProto:
    name: str = ""
    dims: List[int] = field(default_factory=list)
    data_type: int = F32
    array: Optional[np.ndarray] = None  # storage-typed values (fp16 as float16, bf16 as uint16 bit patterns)

    @staticmethod
    def parse(buf) -> "TensorProto":
        t = TensorProto()
        raw = None
        f32, i32, i64, f64, u64 = [], [], [], [], []
        for no, wt, v in _fields(buf):
            if no == 1: t.dims += _packed_ints(wt, v)
            elif no == 2: t.data_type = v
            elif no == 4: f32 += _packed_f32(wt, v)
            elif no == 5: i32 += _packed_ints(wt, v)
            elif no == 7: i64 += _packed_ints(wt, v)
            elif no == 8: t.name = bytes(v).decode()
            elif no == 9: raw = bytes(v)
            elif no == 10: f64 += list(np.frombuffer(v, dtype="<f8")) if wt == 2 else list(struct.unpack("<d", v))
            elif no == 11: u64 += _packed_ints(wt, v)
            elif no == 14 and v != 0: raise ValueError(f"tensor {t.name}: external data is not supported")
        dt = _NP.get(t.data_type)
        if dt is None:
            raise ValueError(f"tensor {t.name}: ONNX data type {t.data_type} not supported")
        if raw is not None:
            arr = np.frombuffer(raw, dtype=np.dtype(dt).newbyteorder("<")).astype(dt, copy=True)
        elif t.data_type in (F16, BF16):  # 16-bit patterns travel in int32_data
            arr = np.array(i32, dtype=np.int64).astype(np.uint16)
            arr = arr.view(np.float16) if t.data_type == F16 else arr
        elif t.data_type == F32: arr = np.array(f32, dtype=np.float32)
        elif t.data_type == F64: arr = np.array(f64, dtype=np.float64)
        elif t.data_type == I64: arr = np.array(i64, dtype=np.int64)
        elif t.data_type == U32: arr = np.array(u64, dtype=np.uint32)
        else: arr = np.array(i32, dtype=np.int64).astype(dt)
        t.array = arr.reshape(t.dims) if t.dims else arr.reshape(())
        return t

    def encode(self) -> bytes:
        out = b"".join(_key(1, 0) + _enc_varint(d) for d in self.dims)
        out += _key(2, 0) + _enc_varint(self.data_type)
        out += _ld(8, self.name.encode())
        out += _ld(9, np.ascontiguousarray(self.array).astype(_NP[self.data_type], copy=False).tobytes())
        return out


@dataclass
class ValueInfo:
    name: str = ""
    elem_type: int = F32
    dims: List[int] = field(default_factory=list)  # dim_param / missing -> 0 (lowered to 1 by the stub)

    @staticmethod
    def parse(buf) -> "ValueInfo":
        vi = ValueInfo()
        for no, _, v in _fields(buf):
            if no == 1: vi.name = bytes(v).decode()
            elif no == 2:
                for n2, _, v2 in _fields(v):
                    if n2 != 1: continue  # TypeProto.tensor_type
                    for n3, _, v3 in _fields(v2):
                        if n3 == 1: vi.elem_type = v3
                        elif n3 == 2:  # TensorShapeProto
                            for n4, _, v4 in _fields(v3):
                                if n4 != 1: continue
                                val = 0
                                for n5, _, v5 in _fields(v4):
                                    if n5 == 1: val = _sint64(v5)
                                vi.dims.append(val)
        return vi

    def encode(self) -> bytes:
        shape = b"".join(_ld(1, _key(1, 0) + _enc_varint(d)) for d in self.dims)
        tensor_type = _key(1, 0) + _enc_varint(self.elem_type) + _ld(2, shape)
        return _ld(1, self.name.encode()) + _ld(2, _ld(1, tensor_type))


@dataclass
class Node:
    op_type: str = ""
    inputs: List[str] = field(default_factory=list)
    outputs: List[str] = field(default_factory=list)
    name: str = ""
    attrs: Dict[str, Any] = field(default_factory=dict)  # int | float | bytes | list | TensorProto
    domain: str = ""  # operator set of the node: "" = the default ONNX domain, "com.microsoft" for MatMulNBits

    @staticmethod
    def parse(buf) -> "Node":
        nd = Node()
        for no, _, v in _fields(buf):
            if no == 1: nd.inputs.append(bytes(v).decode())
            elif no == 2: nd.outputs.append(bytes(v).decode())
            elif no == 3: nd.name = bytes(v).decode()
            elif no == 4: nd.op_type = bytes(v).decode()
            elif no == 5:
                k, val = Node._attr(v)
                nd.attrs[k] = val
            elif no == 7: nd.domain = bytes(v).decode()
        return nd

    @staticmethod
    def _attr(buf):
        name, kind = "", 0
        f = i = s = t = None
        floats, ints, strings = [], [], []
        for no, wt, v in _fields(buf):
            if no == 1: name = bytes(v).decode()
            elif no == 2: f = struct.unpack("<f", v)[0]
            elif no == 3: i = _sint64(v)
            elif no == 4: s = bytes(v)
            elif no == 5: t = TensorProto.parse(v)
            elif no == 7: floats += _packed_f32(wt, v)
            elif no == 8: ints += _packed_ints(wt, v)
            elif no == 9: strings.append(bytes(v))
            elif no == 20: kind = v
        # AttributeProto.AttributeType: 1 FLOAT 2 INT 3 STRING 4 TENSOR 6 FLOATS 7 INTS 8 STRINGS
        val = {1: f, 2: i, 3: s, 4: t, 6: floats, 7: ints, 8: strings}.get(kind)
        if kind == 0:  # writers that omit `type`: take whichever member is present
            val = next((x for x in (t, s, f, i) if x is not None), ints or floats or strings)
        if kind not in (0, 1, 2, 3, 4, 6, 7, 8):
            raise ValueError(f"attribute {name}: type {kind} (graph / sparse tensor) not supported")
        return name, val

    def encode(self) -> bytes:
        out = b"".join(_ld(1, x.encode()) for x in self.inputs) + b"".join(_ld(2, x.encode()) for x in self.outputs)
        out += _ld(3, self.name.encode()) + _ld(4, self.op_type.encode())
        for k, v in self.attrs.items():
            a = _ld(1, k.encode())
            if isinstance(v, bool) or isinstance(v, (int, np.integer)): a += _key(3, 0) + _enc_varint(int(v)) + _key(20, 0) + _enc_varint(2)
            elif isinstance(v, float): a += _key(2, 5) + struct.pack("<f", v) + _key(20, 0) + _enc_varint(1)
            elif isinstance(v, (bytes, str)): a += _ld(4, v.encode() if isinstance(v, str) else v) + _key(20, 0) + _enc_varint(3)
            elif isinstance(v, TensorProto): a += _ld(5, v.encode()) + _key(20, 0) + _enc_varint(4)
            elif len(v) and isinstance(v[0], float): a += b"".join(_key(7, 5) + struct.pack("<f", x) for x in v) + _key(20, 0) + _enc_varint(6)
            else: a += _ld(8, b"".join(_enc_varint(int(x)) for x in v)) + _key(20, 0) + _enc_varint(7)
            out += _ld(5, a)
        if self.domain:  # (default-domain nodes carry no field 7: their bytes are what they always were)
            out += _ld(7, self.domain.encode())
        return out


@dataclass
class Graph:
    nodes: List[Node] = field(default_factory=list)
    initializers: List[TensorProto] = field(default_factory=list)
    inputs: List[ValueInfo] = field(default_factory=list)
    outputs: List[ValueInfo] = field(default_factory=list)
    name: str = "graph"

    @staticmethod
    def parse(buf) -> "Graph":
        g = Graph()
        for no, _, v in _fields(buf):
            if no == 1: g.nodes.append(Node.parse(v))
            elif no == 2: g.name = bytes(v).decode()
            elif no == 5: g.initializers.append(TensorProto.parse(v))
            elif no == 11: g.inputs.append(ValueInfo.parse(v))
            elif no == 12: g.outputs.append(ValueInfo.parse(v))
        return g

    def encode(self) -> bytes:
        return (b"".join(_ld(1, n.encode()) for n in self.nodes) + _ld(2, self.name.encode()) +
                b"".join(_ld(5, t.encode()) for t in self.initializers) +
                b"".join(_ld(11, v.encode()) for v in self.inputs) + b"".join(_ld(12, v.encode()) for v in self.outputs))


@dataclass
class Model:
    graph: Graph = field(default_factory=Graph)
    ir_version: int = 8
    opset: int = 17


def load_model(src) -> Model:
    """`src`: path, bytes or an already parsed Model."""
    if isinstance(src, Model):
        return src
    if isinstance(src, str):
        with open(src, "rb") as f:
            src = f.read()
    m = Model()
    for no, _, v in _fields(src):
        if no == 1: m.ir_version = v
        elif no == 7: m.graph = Graph.parse(v)
        elif no == 8:
            fields = list(_fields(v))
            if any(n2 == 1 and bytes(v2) not in (b"", b"ai.onnx") for n2, _, v2 in fields):
                continue  # another domain's operator set (com.microsoft): its version does not change the default opset
            for n2, _, v2 in fields:
                if n2 == 2: m.opset = v2
    return m


MS_DOMAIN = "com.microsoft"


def save_model(m: Model) -> bytes:
    opset = _ld(1, b"") + _key(2, 0) + _enc_varint(m.opset)
    out = _key(1, 0) + _enc_varint(m.ir_version) + _ld(2, b"infinitensor_b200") + _ld(7, m.graph.encode()) + _ld(8, opset)
    if any(nd.domain == MS_DOMAIN for nd in m.graph.nodes):  # the contrib operator set, only when a node uses it
        out += _ld(8, _ld(1, MS_DOMAIN.encode()) + _key(2, 0) + _enc_varint(1))
    return out


# ------------------------------------------------------------------------------------------------ lowering
class OnnxStub:
    """Mirror of pyinfinitensor.onnx.OnnxStub for the operators this backend implements: builds the graph through
    `handler`, allocates (`data_malloc`) and uploads the initializers.  `inputs` / `outputs` map ONNX names to tensors."""

    def __init__(self, model, runtime=None, handler=None, use_naive_allocator: bool = False, upload: bool = True):
        if handler is None:
            from . import backend
            handler = backend.GraphHandler(runtime)
        self.handler = handler
        self.model = load_model(model)
        self.inputs: Dict[str, Any] = {}
        self.outputs: Dict[str, Any] = {}
        self.tensors: Dict[str, Any] = {}
        self._data: Dict[str, TensorProto] = {}      # constants materialised as weight tensors (uploaded by init())
        self._consts: Dict[str, Any] = {}              # every compile-time constant: name -> (ndarray, ONNX dtype)
        self.folded: List[str] = []                    # op types evaluated at load time, in order (introspection / tests)
        self.lowered_nodes: List[Node] = []            # the nodes that reached the handler, in topological order
        self.use_naive_allocator = use_naive_allocator
        self._build()
        if upload:  # (False: build and plan only, e.g. on the planning runtime of the CPU tests)
            self.init()

    # -- the reference's entry points (onnx.py:1138-1160 region)
    def init(self):
        self.handler.data_malloc(self.use_naive_allocator) if self.use_naive_allocator else self.handler.data_malloc()
        for name, proto in self._data.items():
            self.tensors[name].copyin_numpy(np.ascontiguousarray(proto.array))

    def to_onnx(self, name: str = "") -> bytes:
        """The loaded model back as ONNX bytes, constant subgraphs already folded (reference `OnnxStub.to_onnx`, onnx.py:1138)."""
        used = {x for nd in self.lowered_nodes for x in nd.inputs} | set(self.outputs)
        inits = [TensorProto(n, list(a.shape), dt, a) for n, (a, dt) in self._consts.items() if n in used]
        g = self.model.graph
        return save_model(Model(Graph(list(self.lowered_nodes), inits, [v for v in g.inputs if v.name in self.inputs], list(g.outputs),
                                      name or g.name), self.model.ir_version, self.model.opset))

    def optimize(self): self.handler.optimize()
    def tune(self): self.handler.tune()
    def run(self): self.handler.run()
    def run_with_cudagraph(self): self.handler.run_with_cudagraph()
    def get_perf_time(self): return self.handler.get_perf_time()

    # -- helpers
    def _const(self, name) -> Optional[np.ndarray]:
        c = self._consts.get(name)
        return None if c is None else c[0]

    def _ints(self, node, idx, attr=None, required=False):
        if len(node.inputs) > idx and node.inputs[idx]:
            c = self._const(node.inputs[idx])
            if c is None:
                raise NotImplementedError(f"{node.op_type} {node.name}: input {idx} must be a constant (no dynamic shapes)")
            return [int(x) for x in np.asarray(c).reshape(-1)]
        if attr is not None and attr in node.attrs:
            return [int(x) for x in node.attrs[attr]]
        if required:
            raise ValueError(f"{node.op_type} {node.name}: missing `{attr}`")
        return None

    def _set_const(self, name, arr, dtype=None):
        arr = np.asarray(arr)
        if dtype is None:
            dtype = next((k for k, v in _NP.items() if k != BF16 and np.dtype(v) == arr.dtype), None)
            if dtype is None:
                raise NotImplementedError(f"constant {name}: numpy dtype {arr.dtype} has no ONNX code here")
        self._consts[name] = (arr, dtype)

    def _operand(self, name):
        """Tensor for an operator input; a compile-time constant becomes a weight tensor on first use."""
        t = self.tensors.get(name)
        if t is None:
            arr, dtype = self._consts[name]
            if arr.ndim == 0:
                arr = arr.reshape(1)  # scalars travel as [1] (same broadcasting; rank-0 device tensors are avoided)
            t = self.handler.tensor(list(arr.shape), dtype)
            t.set_weight()
            self.tensors[name] = t
            self._data[name] = TensorProto(name, list(arr.shape), dtype, arr)
        return t

    def _build(self):
        g, h, T = self.model.graph, self.handler, self.tensors
        for init in g.initializers:
            self._set_const(init.name, init.array, init.data_type)
        for vi in g.inputs:
            if vi.name not in self._consts:
                T[vi.name] = h.tensor([d if d > 0 else 1 for d in vi.dims], vi.elem_type)
                T[vi.name].set_input()
                self.inputs[vi.name] = T[vi.name]
        # topological order over tensor availability (the file order of exported models is not guaranteed)
        known = set(T) | set(self._consts)
        pending = list(range(len(g.nodes)))
        order = []
        while pending:
            rest = []
            for i in pending:
                if all(x in known or x == "" for x in g.nodes[i].inputs):
                    order.append(i)
                    known.update(g.nodes[i].outputs)
                else:
                    rest.append(i)
            if len(rest) == len(pending):
                bad = g.nodes[rest[0]]
                raise ValueError(f"ONNX graph has a cycle or a missing input near {bad.op_type} {bad.name}: "
                                 f"{[x for x in bad.inputs if x and x not in known]}")
            pending = rest
        for i in order:
            nd = g.nodes[i]
            if not self._fold(nd):
                self._lower(nd)
                self.lowered_nodes.append(nd)
        for vo in g.outputs:
            self._operand(vo.name).set_output()
            self.outputs[vo.name] = T[vo.name]

    # ---- load-time evaluation of constant subgraphs (what the reference delegates to onnxsim)
    def _fold(self, nd: Node) -> bool:
        op, a = nd.op_type, nd.attrs
        if op == "Constant":
            v = a.get("value")
            if isinstance(v, TensorProto):
                self._set_const(nd.outputs[0], v.array, v.data_type)
            elif "value_int" in a: self._set_const(nd.outputs[0], np.array(a["value_int"], np.int64))
            elif "value_ints" in a: self._set_const(nd.outputs[0], np.array(a["value_ints"], np.int64))
            elif "value_float" in a: self._set_const(nd.outputs[0], np.array(a["value_float"], np.float32))
            elif "value_floats" in a: self._set_const(nd.outputs[0], np.array(a["value_floats"], np.float32))
            else: raise NotImplementedError("Constant: unsupported value form")
            return True
        if op == "Shape":  # static shapes: the shape of ANY tensor is known now
            src = nd.inputs[0]
            shp = list(self._consts[src][0].shape) if src in self._consts else list(self.tensors[src].shape())
            n = len(shp)
            st, en = a.get("start", 0), a.get("end", n)
            st, en = (st + n if st < 0 else st), (en + n if en < 0 else en)
            self._set_const(nd.outputs[0], np.array(shp[max(st, 0):min(en, n)], np.int64))
            self.folded.append(op)
            return True
        fn = self._FOLD.get(op)
        if fn is None or not all(x == "" or x in self._consts for x in nd.inputs):
            return False
        ins = [None if x == "" else self._consts[x][0] for x in nd.inputs]
        dts = [None if x == "" else self._consts[x][1] for x in nd.inputs]
        out = fn(ins, a)
        outs = out if isinstance(out, list) else [out]
        for name, arr in zip(nd.outputs, outs):
            arr = np.asarray(arr)
            keep = op not in ("Cast", "Equal", "Less", "Greater", "Not", "ConstantOfShape", "Range") and dts and dts[0] is not None \
                and np.dtype(_NP[dts[0]]) == arr.dtype
            self._set_const(name, arr, dts[0] if keep else (a["to"] if op == "Cast" else None))
        self.folded.append(op)
        return True

    @staticmethod
    def _slice_np(ins, a):
        x = ins[0]
        starts = [int(v) for v in (ins[1] if len(ins) > 1 and ins[1] is not None else a["starts"])]
        ends = [int(v) for v in (ins[2] if len(ins) > 2 and ins[2] is not None else a["ends"])]
        axes = [int(v) for v in (ins[3] if len(ins) > 3 and ins[3] is not None else a.get("axes", range(len(starts))))]
        steps = [int(v) for v in (ins[4] if len(ins) > 4 and ins[4] is not None else [1] * len(starts))]
        sl = [slice(None)] * x.ndim
        for s0, e0, ax, st in zip(starts, ends, axes, steps):
            sl[ax] = slice(s0, e0, st)  # numpy clamps out-of-range bounds exactly like ONNX Slice
        return x[tuple(sl)]

    @staticmethod
    def _div_np(a, b):
        if np.issubdtype(np.asarray(a).dtype, np.integer):
            return np.trunc(np.asarray(a, np.float64) / np.asarray(b, np.float64)).astype(np.asarray(a).dtype)  # C-style
        return a / b

    _FOLD = {
        "Identity": lambda i, a: i[0],
        "Gather": lambda i, a: np.take(i[0], np.asarray(i[1], np.int64), axis=a.get("axis", 0)),
        "Unsqueeze": lambda i, a: np.expand_dims(i[0], tuple(int(v) for v in (i[1] if len(i) > 1 else a["axes"]))),
        "Squeeze": lambda i, a: np.squeeze(i[0], tuple(int(v) for v in (i[1] if len(i) > 1 and i[1] is not None else a["axes"]))
                                           if (len(i) > 1 and i[1] is not None) or "axes" in a else None),
        "Concat": lambda i, a: np.concatenate([np.atleast_1d(v) for v in i], axis=a["axis"]),
        "Cast": lambda i, a: i[0].astype(_NP[a["to"]]),
        "Slice": lambda i, a: OnnxStub._slice_np(i, a),
        "Add": lambda i, a: i[0] + i[1], "Sub": lambda i, a: i[0] - i[1], "Mul": lambda i, a: i[0] * i[1],
        "Div": lambda i, a: OnnxStub._div_np(i[0], i[1]),
        "Neg": lambda i, a: -i[0], "Sqrt": lambda i, a: np.sqrt(i[0]),
        "Min": lambda i, a: np.minimum(i[0], i[1]), "Max": lambda i, a: np.maximum(i[0], i[1]),
        "Equal": lambda i, a: np.equal(i[0], i[1]), "Less": lambda i, a: np.less(i[0], i[1]),
        "Greater": lambda i, a: np.greater(i[0], i[1]), "Not": lambda i, a: np.logical_not(i[0]),
        "Where": lambda i, a: np.where(i[0], i[1], i[2]),
        "Reshape": lambda i, a: i[0].reshape([i[0].shape[k] if v == 0 else int(v) for k, v in enumerate(i[1])]),
        "Expand": lambda i, a: np.broadcast_to(i[0], np.broadcast_shapes(i[0].shape, tuple(int(v) for v in i[1]))).copy(),
        "Transpose": lambda i, a: np.transpose(i[0], a.get("perm")),
        "ReduceProd": lambda i, a: np.prod(i[0], axis=tuple(a["axes"]) if "axes" in a else None, keepdims=bool(a.get("keepdims", 1))),
        "ConstantOfShape": lambda i, a: np.full([int(v) for v in i[0]], a["value"].array.reshape(-1)[0] if "value" in a else np.float32(0),
                                                dtype=a["value"].array.dtype if "value" in a else np.float32),
        "Range": lambda i, a: np.arange(i[0], i[1], i[2]).astype(np.asarray(i[0]).dtype),
    }

    _UNARY = {"Relu": "relu", "Silu": "silu", "Gelu": "gelu", "Sigmoid": "sigmoid", "Tanh": "tanh", "Erf": "erf",
              "Abs": "abs", "Sqrt": "sqrt", "Neg": "neg", "HardSigmoid": "hardSigmoid", "HardSwish": "hardSwish",
              "Identity": "identity", "Exp": "exp"}
    _BINARY = {"Add": "add", "Sub": "sub", "Mul": "mul", "Div": "div", "Pow": "pow", "Min": "min", "Max": "max",
               "Less": "less", "Equal": "equal", "Greater": "greater"}
    _ALLREDUCE = {"AllReduceSum": "allReduceSum", "AllReduceProd": "allReduceProd", "AllReduceMin": "allReduceMin",
                  "AllReduceMax": "allReduceMax", "AllReduceAvg": "allReduceAvg"}

    def _lower(self, nd: Node):
        h, T, op, a = self.handler, self.tensors, nd.op_type, nd.attrs
        I = lambda k: self._operand(nd.inputs[k])
        out0 = nd.outputs[0] if nd.outputs else None
        if op in self._UNARY:
            T[out0] = getattr(h, self._UNARY[op])(I(0), None)
        elif op in self._BINARY:
            T[out0] = getattr(h, self._BINARY[op])(I(0), I(1), None)
        elif op in self._ALLREDUCE:
            T[out0] = getattr(h, self._ALLREDUCE[op])(I(0), None)
        elif op == "Dropout":
            T[out0] = h.identity(I(0), None)
        elif op == "MatMul":
            T[out0] = h.matmul(I(0), I(1), None, False, False, None, 0)
        elif op == "MatMulNBits":
            # com.microsoft MatMulNBits: A, B, scales, [zero_points], [g_idx], [bias]; accuracy_level is read and ignored
            opt = [I(i) if len(nd.inputs) > i and nd.inputs[i] else None for i in (3, 4, 5)]
            T[out0] = h.matMulNBits(I(0), I(1), I(2), opt[0], None, a["K"], a["N"], a["block_size"], bits=a.get("bits", 4),
                                    g_idx=opt[1], bias=opt[2])
        elif op == "Gemm":
            if a.get("alpha", 1.0) != 1.0 or a.get("beta", 1.0) != 1.0:
                raise NotImplementedError("Gemm: alpha / beta other than 1 are not supported (reference onnx.py:298-300)")
            bias = I(2) if len(nd.inputs) > 2 and nd.inputs[2] else None
            T[out0] = h.matmul(I(0), I(1), None, a.get("transA", 0) == 1, a.get("transB", 0) == 1, bias, 0)
        elif op == "Conv":
            d, p, s = a.get("dilations", [1, 1]), list(a.get("pads", [0, 0, 0, 0])), a.get("strides", [1, 1])
            if a.get("group", 1) != 1 and I(1).shape()[1] * a["group"] != I(0).shape()[1]:
                raise ValueError("Conv: `group` does not match the filter's channel count")
            x = I(0)
            if p[0] != p[2] or p[1] != p[3]:  # asymmetric padding: explicit Pad on H, W
                x = h.pad(x, None, p, [-2, -1])
                p = [0, 0, 0, 0]
            y = h.conv(x, I(1), None, p[0], p[1], s[0], s[1], d[0], d[1])
            if len(nd.inputs) > 2 and nd.inputs[2]:
                b = I(2)
                y = h.add(y, h.reshape(b, None, [1, int(np.prod(b.shape())), 1, 1]), None)
            T[out0] = y
        elif op == "BatchNormalization":
            T[out0] = h.batchNormalization(I(0), None, I(3), I(4), I(1), I(2), float(a.get("momentum", 0.9)),
                                           float(a.get("epsilon", 1e-5)), a.get("training_mode", 0) != 0)
        elif op == "LayerNormalization":
            bias = I(2) if len(nd.inputs) > 2 and nd.inputs[2] else None
            T[out0] = h.layerNormalization(I(0), I(1), None, bias, float(a.get("epsilon", 1e-5)), a.get("axis", -1),
                                           a.get("stash_type", 1))
        elif op == "RMSNorm":
            T[out0] = h.RMSNorm(I(0), I(1), None)
        elif op == "RoPE":  # optional int attribute dim_head and optional input 2, inv_freq (extensions; absent = the reference's)
            kw = {"inv_freq": I(2)} if len(nd.inputs) > 2 and nd.inputs[2] else {}
            if kw and not getattr(h, "rope_inv_freq", False):
                raise NotImplementedError(f"RoPE {nd.name}: {type(h).__name__} does not execute an inv_freq table")
            if "dim_head" in a and int(a["dim_head"]) != 128:
                if int(a["dim_head"]) not in getattr(h, "head_widths", (128,)):
                    raise NotImplementedError(f"RoPE {nd.name}: {type(h).__name__} does not execute dim_head {a['dim_head']}")
                T[out0] = h.RoPE(I(0), I(1), None, int(a["dim_head"]), **kw)
            else:
                T[out0] = h.RoPE(I(0), I(1), None, **kw)
        elif op == "AttentionKVCache":  # optional inputs 6, 7 (extension): k_scale / v_scale of FP8 E4M3 caches
            kw = {"k_scale": I(6), "v_scale": I(7)} if len(nd.inputs) > 6 else {}
            if int(a.get("window", 0)):  # int attribute window (extension): sliding-window attention, absent = 0 = none
                if not getattr(h, "sliding_window", False):
                    raise NotImplementedError(f"AttentionKVCache {nd.name}: {type(h).__name__} has no sliding window")
                kw["window"] = int(a["window"])
            if int(a.get("rolling", 0)):  # int attribute rolling (extension): the caches are a ring, absent = 0 = linear
                if not getattr(h, "rolling_cache", False):
                    raise NotImplementedError(f"AttentionKVCache {nd.name}: {type(h).__name__} has no rolling KV cache")
                kw["rolling"] = True
            T[out0] = h.attentionKVCache(I(0), I(1), I(2), I(3), I(4), I(5), None, **kw)
        elif op in ("MaxPool", "AveragePool"):
            k = a["kernel_shape"]
            d, p, s = a.get("dilations", [1, 1]), list(a.get("pads", [0, 0, 0, 0])), a.get("strides", [1, 1])
            x = I(0)
            if p[0] != p[2] or p[1] != p[3]:
                x = h.pad(x, None, p, [-2, -1])
                p = [0, 0, 0, 0]
            fn = h.maxPool if op == "MaxPool" else h.avgPool
            T[out0] = fn(x, None, k[0], k[1], d[0], d[1], p[0], p[1], s[0], s[1], a.get("ceil_mode", 0))
        elif op == "GlobalAveragePool":
            hh, ww = I(0).shape()[2:4]
            T[out0] = h.avgPool(I(0), None, hh, ww, 1, 1, 0, 0, 1, 1, 0)
        elif op == "Softmax":
            T[out0] = h.softmax(I(0), None, a.get("axis", -1))
        elif op == "Flatten":
            T[out0] = h.flatten(I(0), None, a.get("axis", 1))
        elif op == "Transpose":
            perm = a.get("perm") or list(range(len(I(0).shape())))[::-1]
            T[out0] = h.transpose(I(0), None, [int(x) for x in perm])
        elif op == "DepthToSpace":  # onnx.py:656-670
            mode = a.get("mode", b"DCR")
            T[out0] = h.depthToSpace(I(0), None, int(a["blocksize"]), mode.decode() if isinstance(mode, bytes) else mode)
        elif op == "Reshape":
            shape = self._ints(nd, 1, "shape", required=True)
            src = I(0).shape()
            shape = [src[i] if v == 0 and not a.get("allowzero", 0) else v for i, v in enumerate(shape)]
            if -1 in shape:
                known = int(np.prod([v for v in shape if v != -1])) or 1
                shape[shape.index(-1)] = int(np.prod(src)) // known
            T[out0] = h.reshape(I(0), None, shape)
        elif op == "Squeeze":
            axes = self._ints(nd, 1, "axes")
            if axes is None:
                axes = [i for i, v in enumerate(I(0).shape()) if v == 1]
            T[out0] = h.squeeze(I(0), None, axes)
        elif op == "Unsqueeze":
            T[out0] = h.unsqueeze(I(0), None, self._ints(nd, 1, "axes", required=True))
        elif op == "Concat":
            T[out0] = h.concat([self._operand(x) for x in nd.inputs], None, a["axis"])
        elif op == "Split":
            axis = a.get("axis", 0)
            split = self._ints(nd, 1, "split")
            outs = h.split(I(0), None, axis, split if split is not None else len(nd.outputs))
            for name, t in zip(nd.outputs, outs):
                T[name] = t
        elif op == "Gather":
            T[out0] = h.gather(I(0), I(1), None, a.get("axis", 0))
        elif op in ("ReduceMean", "ReduceSum"):
            if op == "ReduceSum" and "communicator" in a:
                T[out0] = h.allReduceSum(I(0), None)
            else:
                axes = self._ints(nd, 1, "axes")
                fn = h.reduceMean if op == "ReduceMean" else h.reduceSum
                T[out0] = fn(I(0), None, axes, a.get("keepdims", 1) != 0)
        elif op == "Slice":
            starts, ends = self._ints(nd, 1, "starts", required=True), self._ints(nd, 2, "ends", required=True)
            lim = np.iinfo(np.int32)
            clamp = lambda v: [max(lim.min, min(lim.max, int(x))) for x in v]
            T[out0] = h.slice(I(0), None, clamp(starts), clamp(ends), self._ints(nd, 3, "axes"), self._ints(nd, 4, "steps"))
        elif op == "Pad":
            if a.get("mode", b"constant") not in (b"constant", "constant"):
                raise NotImplementedError("Pad: only constant mode")
            T[out0] = h.pad(I(0), None, self._ints(nd, 1, "pads", required=True), self._ints(nd, 3, "axes"))
        elif op == "Cast":
            T[out0] = h.cast(I(0), None, a["to"])
        elif op == "Expand":
            T[out0] = h.expand(I(0), None, self._ints(nd, 1, "shape", required=True))
        elif op == "Where":
            cond, alt = self._const(nd.inputs[0]), self._const(nd.inputs[2])
            if cond is not None and alt is not None and alt.size == 1 and (np.isneginf(alt).all() or (alt < -3e38).all()):
                # a constant mask selecting between x and a single -inf (causal masks): an additive 0 / -inf bias instead of a
                # three-operand select (the reference's rewrite, onnx.py:1055-1081)
                name = nd.inputs[0] + "_alt"
                if name not in self._consts:
                    self._set_const(name, np.where(cond, 0, -np.inf).astype(alt.dtype), self._consts[nd.inputs[2]][1])
                T[out0] = h.add(I(1), self._operand(name), None)
            else:
                T[out0] = h.where(I(1), I(2), I(0), None)
        elif op == "AllGather":
            outs = h.allGather(I(0), None, len(nd.outputs))
            for name, t in zip(nd.outputs, outs):
                T[name] = t
        else:
            raise NotImplementedError(f'Unsupported operator "{op}" (no B200 kernel behind it)')


# ------------------------------------------------------------------------------------------------ export
class _ExportTensor:
    """Tensor of the wrapped handler + the ONNX name it is exported under; records uploaded weight values."""

    def __init__(self, exporter, inner, name):
        self._x, self.inner, self.name = exporter, inner, name

    def shape(self): return self.inner.shape()
    def dtype(self): return self.inner.dtype()
    def fuid(self): return self.inner.fuid() if hasattr(self.inner, "fuid") else id(self.inner)

    def set_weight(self):
        self.inner.set_weight()
        self._x._weights[self.name] = None

    def set_input(self):
        self.inner.set_input()
        self._x._inputs.append(self)

    def set_output(self):
        self.inner.set_output()
        self._x._outputs.append(self)

    def copyin_numpy(self, arr):
        if self.name in self._x._weights:
            self._x._weights[self.name] = np.array(arr, copy=True)
        else:
            self.inner.copyin_numpy(arr)

    def copyout_numpy(self): return self.inner.copyout_numpy()


class OnnxExporter:
    """Handler decorator that records every call as an ONNX node (the direction of the reference's `OnnxStub.to_onnx`,
    onnx.py:1138-1482): build any graph through it -- e.g. `graphs.build_llama_decode(OnnxExporter(h), cfg)` -- then
    `model()` / `save()` give the ONNX file `OnnxStub` reads back.  Shapes come from the wrapped handler."""

    def __init__(self, inner):
        self.inner = inner
        self.nodes: List[Node] = []
        self._weights: Dict[str, Optional[np.ndarray]] = {}
        self._inputs: List[_ExportTensor] = []
        self._outputs: List[_ExportTensor] = []
        self._all: List[_ExportTensor] = []
        self._by_inner: Dict[Any, _ExportTensor] = {}
        self._const_protos: Dict[str, TensorProto] = {}
        self._n = 0

    @staticmethod
    def _tid(t):
        return ("id", t.fuid()) if hasattr(t, "fuid") else ("py", id(t))

    def _wrap(self, t, prefix="t"):
        k = self._tid(t)
        if k in self._by_inner:  # an output tensor the builder created up front and passed in
            return self._by_inner[k]
        w = _ExportTensor(self, t, f"{prefix}{self._n}")
        self._n += 1
        self._all.append(w)
        self._by_inner[k] = w
        return w

    def tensor(self, dims, dtype):
        return self._wrap(self.inner.tensor(dims, dtype), "v")

    def _const(self, values, dtype=I64):
        arr = np.asarray(values, dtype=_NP[dtype])
        w = _ExportTensor(self, None, f"c{self._n}")
        self._n += 1
        self._weights[w.name] = arr
        self._const_protos[w.name] = TensorProto(w.name, list(arr.shape), dtype, arr)
        return w.name

    def _emit(self, op, ins, inner_out, attrs=None, extra_inputs=()):
        outs = inner_out if isinstance(inner_out, (list, tuple)) else [inner_out]
        wrapped = [self._wrap(o) for o in outs]
        names = [("" if t is None else t.name) for t in ins] + list(extra_inputs)
        self.nodes.append(Node(op, names, [w.name for w in wrapped], f"{op}_{len(self.nodes)}", dict(attrs or {})))
        return wrapped if isinstance(inner_out, (list, tuple)) else wrapped[0]

    @staticmethod
    def _in(t): return None if t is None else t.inner

    # ---- operators: same signatures as backend.GraphHandler
    def matmul(self, a, b, y, transA, transB, bias, act, matmul_compute_type="default"):
        r = self.inner.matmul(a.inner, b.inner, self._in(y), transA, transB, self._in(bias), act)
        if not transA and not transB and bias is None:
            return self._emit("MatMul", [a, b], r)
        return self._emit("Gemm", [a, b] + ([bias] if bias is not None else []), r,
                          {"transA": int(bool(transA)), "transB": int(bool(transB))})

    def matMulNBits(self, a, b, scales, zero_points, y, K, N, block_size, bits=4, g_idx=None, bias=None):
        r = self.inner.matMulNBits(a.inner, b.inner, scales.inner, self._in(zero_points), self._in(y), K, N, block_size, bits,
                                   self._in(g_idx), self._in(bias))
        ins = [a, b, scales, zero_points, g_idx, bias]
        while ins[-1] is None:  # trailing absent optional inputs are omitted, inner ones named ""
            ins.pop()
        out = self._emit("MatMulNBits", ins, r, {"K": int(K), "N": int(N), "bits": int(bits), "block_size": int(block_size)})
        self.nodes[-1].domain = MS_DOMAIN
        return out

    def conv(self, x, w, y, ph, pw, sh, sw, dh, dw):
        r = self.inner.conv(x.inner, w.inner, self._in(y), ph, pw, sh, sw, dh, dw)
        return self._emit("Conv", [x, w], r, {"pads": [ph, pw, ph, pw], "strides": [sh, sw], "dilations": [dh, dw],
                                              "group": x.shape()[1] // w.shape()[1]})

    def batchNormalization(self, x, y, mean, var, scale, bias, momentum, eps, training):
        r = self.inner.batchNormalization(x.inner, self._in(y), mean.inner, var.inner, scale.inner, bias.inner, momentum, eps,
                                          training)
        return self._emit("BatchNormalization", [x, scale, bias, mean, var], r,
                          {"momentum": float(momentum), "epsilon": float(eps), "training_mode": int(bool(training))})

    def layerNormalization(self, x, scale, y, bias, eps, axis, stash_type):
        r = self.inner.layerNormalization(x.inner, scale.inner, self._in(y), self._in(bias), eps, axis, stash_type)
        return self._emit("LayerNormalization", [x, scale] + ([bias] if bias is not None else []), r,
                          {"epsilon": float(eps), "axis": int(axis), "stash_type": int(stash_type)})

    def RMSNorm(self, x, w, y): return self._emit("RMSNorm", [x, w], self.inner.RMSNorm(x.inner, w.inner, self._in(y)))
    def RoPE(self, pos, x, y, dim_head=128, inv_freq=None):
        # the attribute only when it is not the reference's 128, the third input only when given: older files stay as they were
        extra = [] if dim_head == 128 else [int(dim_head)]
        kw = {} if inv_freq is None else {"inv_freq": inv_freq.inner}
        return self._emit("RoPE", [pos, x] + ([inv_freq] if inv_freq is not None else []),
                          self.inner.RoPE(pos.inner, x.inner, self._in(y), *extra, **kw), {"dim_head": extra[0]} if extra else None)

    def attentionKVCache(self, kc, vc, q, k, v, pos, y, k_scale=None, v_scale=None, window=0, rolling=False):
        # the FP8 caches' scales, the window and the ring only when given: every other export stays as it was
        scales = [] if k_scale is None else [k_scale, v_scale]
        kw = {"k_scale": k_scale.inner, "v_scale": v_scale.inner} if scales else {}
        attrs = {}
        if window:
            kw["window"] = attrs["window"] = int(window)
        if rolling:
            if not getattr(self.inner, "rolling_cache", False):
                raise NotImplementedError(f"AttentionKVCache: {type(self.inner).__name__} has no rolling KV cache")
            kw["rolling"] = True
            attrs["rolling"] = 1
        r = self.inner.attentionKVCache(kc.inner, vc.inner, q.inner, k.inner, v.inner, pos.inner, self._in(y), **kw)
        return self._emit("AttentionKVCache", [kc, vc, q, k, v, pos] + scales, r, attrs or None)

    def _pool(self, op, fn, x, y, kh, kw, dh, dw, ph, pw, sh, sw, ceil):
        r = fn(x.inner, self._in(y), kh, kw, dh, dw, ph, pw, sh, sw, ceil)
        return self._emit(op, [x], r, {"kernel_shape": [kh, kw], "dilations": [dh, dw], "pads": [ph, pw, ph, pw],
                                       "strides": [sh, sw], "ceil_mode": int(ceil)})

    def maxPool(self, x, y, *a): return self._pool("MaxPool", self.inner.maxPool, x, y, *a)
    def avgPool(self, x, y, *a): return self._pool("AveragePool", self.inner.avgPool, x, y, *a)

    def softmax(self, x, y, axis): return self._emit("Softmax", [x], self.inner.softmax(x.inner, self._in(y), axis), {"axis": int(axis)})
    def flatten(self, x, y, axis): return self._emit("Flatten", [x], self.inner.flatten(x.inner, self._in(y), axis), {"axis": int(axis)})

    def transpose(self, x, y, perm):
        return self._emit("Transpose", [x], self.inner.transpose(x.inner, self._in(y), perm), {"perm": [int(p) for p in perm]})

    def depthToSpace(self, x, y, blocksize, mode):
        return self._emit("DepthToSpace", [x], self.inner.depthToSpace(x.inner, self._in(y), blocksize, mode),
                          {"blocksize": int(blocksize), "mode": mode})

    def reshape(self, x, y, shape):
        r = self.inner.reshape(x.inner, self._in(y), shape)
        return self._emit("Reshape", [x], r, extra_inputs=[self._const(list(shape))])

    def squeeze(self, x, y, axes):
        return self._emit("Squeeze", [x], self.inner.squeeze(x.inner, self._in(y), axes), extra_inputs=[self._const(list(axes))])

    def unsqueeze(self, x, y, axes):
        return self._emit("Unsqueeze", [x], self.inner.unsqueeze(x.inner, self._in(y), axes), extra_inputs=[self._const(list(axes))])

    def concat(self, inputs, y, dim):
        return self._emit("Concat", list(inputs), self.inner.concat([t.inner for t in inputs], self._in(y), dim), {"axis": int(dim)})

    def split(self, x, outputs, axis, numOrRatio):
        inner_outs = None if outputs is None else [self._in(o) for o in outputs]
        r = self.inner.split(x.inner, inner_outs, axis, numOrRatio)
        r = list(r) if isinstance(r, (list, tuple)) else [r]
        if isinstance(numOrRatio, int):
            return self._emit("Split", [x], r, {"axis": int(axis)})
        # ONNX wants element counts; the handler takes ratios -> scale them to the axis length
        n = x.shape()[axis]
        sizes = [n * int(v) // int(sum(numOrRatio)) for v in numOrRatio]
        return self._emit("Split", [x], r, {"axis": int(axis)}, extra_inputs=[self._const(sizes)])

    def gather(self, data, idx, y, axis):
        return self._emit("Gather", [data, idx], self.inner.gather(data.inner, idx.inner, self._in(y), axis), {"axis": int(axis)})

    def _reduce(self, op, fn, x, y, axes, keepdims):
        r = fn(x.inner, self._in(y), axes, keepdims)
        extra = [] if axes is None else [self._const(list(axes))]
        return self._emit(op, [x], r, {"keepdims": int(bool(keepdims))}, extra_inputs=extra)

    def reduceMean(self, x, y, axes, keepdims): return self._reduce("ReduceMean", self.inner.reduceMean, x, y, axes, keepdims)
    def reduceSum(self, x, y, axes, keepdims): return self._reduce("ReduceSum", self.inner.reduceSum, x, y, axes, keepdims)

    def slice(self, x, y, starts, ends, axes, steps):
        r = self.inner.slice(x.inner, self._in(y), starts, ends, axes, steps)
        n = len(starts)
        extra = [self._const(list(starts)), self._const(list(ends)), self._const(list(axes) if axes is not None else list(range(n))),
                 self._const(list(steps) if steps is not None else [1] * n)]
        return self._emit("Slice", [x], r, extra_inputs=extra)

    def pad(self, x, y, pads, axes):
        r = self.inner.pad(x.inner, self._in(y), pads, axes)
        extra = [self._const(list(pads))] + ([] if axes is None else ["", self._const(list(axes))])
        return self._emit("Pad", [x], r, extra_inputs=extra)

    def cast(self, x, y, to): return self._emit("Cast", [x], self.inner.cast(x.inner, self._in(y), to), {"to": int(to)})

    def expand(self, x, y, dims):
        return self._emit("Expand", [x], self.inner.expand(x.inner, self._in(y), dims), extra_inputs=[self._const(list(dims))])

    def where(self, xx, yy, cond, y):
        return self._emit("Where", [cond, xx, yy], self.inner.where(xx.inner, yy.inner, cond.inner, self._in(y)))

    def allGather(self, x, outputs, n):
        inner_outs = None if outputs is None else [self._in(o) for o in outputs]
        return self._emit("AllGather", [x], list(self.inner.allGather(x.inner, inner_outs, n)))

    def __getattr__(self, name):
        # unary / binary / all-reduce families share one shape: (inputs..., output)
        onnx_name = {v: k for k, v in {**OnnxStub._UNARY, **OnnxStub._BINARY, **OnnxStub._ALLREDUCE}.items()}.get(name)
        if onnx_name is None:
            return getattr(self.inner, name)  # data_malloc, run, schedule, ... go straight through

        def call(*args):
            ins = list(args[:-1])
            return self._emit(onnx_name, ins, getattr(self.inner, name)(*[t.inner for t in ins], self._in(args[-1])))
        return call

    # ---- result
    def model(self) -> Model:
        g = Graph(nodes=list(self.nodes))
        consts = self._const_protos
        by_name = {t.name: t for t in self._all}
        for name, arr in self._weights.items():
            if name in consts:
                g.initializers.append(consts[name])
                continue
            t = by_name[name]
            if arr is None:
                arr = np.zeros(t.shape(), dtype=_NP[t.dtype()])
            g.initializers.append(TensorProto(name, list(t.shape()), t.dtype(), np.asarray(arr)))
        g.inputs = [ValueInfo(t.name, t.dtype(), list(t.shape())) for t in self._inputs]
        g.outputs = [ValueInfo(t.name, t.dtype(), list(t.shape())) for t in self._outputs]
        return Model(graph=g)

    def save(self) -> bytes:
        return save_model(self.model())


# ------------------------------------------------------------------------------------------------ model-level passes
def _planning_handler():
    from . import backend
    return backend.GraphHandler(backend.HostPlanRuntime())


def simplify(model, new_handler=None) -> Model:
    """What the reference runs onnxsim for (onnx.py:49-58): the constant subgraphs -- exporter shape arithmetic -- are evaluated
    and removed; their results become initializers.  Shapes come from lowering the model once on a fresh handler from
    `new_handler()` (default: the planning-only runtime, no GPU needed).  Nodes come out in topological order."""
    m = load_model(model)
    stub = OnnxStub(m, handler=(new_handler or _planning_handler)(), upload=False)
    kept = [nd for nd in stub.lowered_nodes]
    used = {x for nd in kept for x in nd.inputs} | {o.name for o in m.graph.outputs}
    inits = [TensorProto(name, list(arr.shape), dt, arr) for name, (arr, dt) in stub._consts.items() if name in used]
    inputs = [ValueInfo(v.name, v.elem_type, [d if d > 0 else 1 for d in v.dims]) for v in m.graph.inputs if v.name not in stub._consts]
    return Model(Graph(kept, inits, inputs, list(m.graph.outputs), m.graph.name), m.ir_version, m.opset)


def tensor_shapes(model, new_handler=None) -> Dict[str, List[int]]:
    """Static shape of every tensor of the model (constants included), from one lowering pass."""
    stub = OnnxStub(load_model(model), handler=(new_handler or _planning_handler)(), upload=False)
    shapes = {name: list(arr.shape) for name, (arr, _) in stub._consts.items()}
    shapes.update({name: list(t.shape()) for name, t in stub.tensors.items()})
    return shapes


def parallel_model(model, world: int, rank: int, new_handler=None) -> Model:
    """Tensor-parallel rewrite of an ONNX model for rank `rank` of `world` -- the job of the reference's
    examples/distributed/parallel_opt.py::parallel_model, on this module's Model classes:

      * a MatMul / Gemm with a constant weight fed by a REPLICATED activation is column-split (per group when a Split of the
        packed result follows within two nodes); its output is sharded on the last axis;
      * fed by an activation sharded on its last axis it is row-split, and a `ReduceSum(communicator=0)` node -- which the
        frontend lowers to AllReduceSum (onnx.py:917-923) -- makes the result replicated again; a Gemm bias is added once, after;
      * the last MatMul (the one producing a graph output) stays replicated, like embeddings, norms and the residual stream;
      * placements flow through unary / binary ops, RoPE (its inv_freq table replicated), Transpose (through the permutation), Split, AttentionKVCache (heads;
        the cache INPUTS shrink on the head axis) and Reshape (the output axis whose row-major prefix product equals the
        sharded input axis' takes the division).
    The model is simplified first, so Reshape targets are plain initializers."""
    m = simplify(model, new_handler)
    if world == 1:
        return m
    for nd in m.graph.nodes:
        if nd.op_type == "MatMulNBits":
            raise NotImplementedError(f"MatMulNBits {nd.name}: tensor-parallel sharding of 4-bit weights is not provided")
    shapes = tensor_shapes(m, new_handler)
    g = m.graph
    consts = {t.name: t for t in g.initializers}
    outputs = {o.name for o in g.outputs}
    inputs = {v.name: v for v in g.inputs}
    place: Dict[str, Any] = {}          # tensor -> sharded axis (int); absent = replicated
    nodes: List[Node] = []
    fresh = [0]

    def shard_array(arr, axis, groups=1):
        axis %= arr.ndim
        n = arr.shape[axis]
        if n % (groups * world):
            raise ValueError(f"axis of {n} elements does not split into {groups} groups x {world} ranks")
        seg = n // groups // world
        view = arr.reshape(arr.shape[:axis] + (groups, n // groups) + arr.shape[axis + 1:])
        return np.ascontiguousarray(np.take(view, range(rank * seg, (rank + 1) * seg), axis=axis + 1)).reshape(
            arr.shape[:axis] + (n // world,) + arr.shape[axis + 1:])

    def new_const(base, arr, dtype):
        fresh[0] += 1
        name = f"{base}@tp{fresh[0]}"
        consts[name] = TensorProto(name, list(arr.shape), dtype, arr)
        return name

    def last_axis(name):
        return len(shapes[name]) - 1

    for nd in g.nodes:  # every rank needs whole KV heads (grouped-query attention may have fewer than `world`)
        if nd.op_type == "AttentionKVCache" and nd.inputs[0] in inputs and inputs[nd.inputs[0]].dims[1] % world:
            raise NotImplementedError(f"AttentionKVCache {nd.name}: {inputs[nd.inputs[0]].dims[1]} KV heads do not split "
                                      f"over {world} ranks")
    unary_like = set(OnnxStub._UNARY) | {"Softmax", "Cast", "Dropout"}
    for idx, nd in enumerate(g.nodes):
        nd = Node(nd.op_type, list(nd.inputs), list(nd.outputs), nd.name, dict(nd.attrs))
        op = nd.op_type
        if op in ("MatMul", "Gemm") and len(nd.inputs) > 1 and nd.inputs[1] in consts and len(shapes[nd.inputs[1]]) == 2:
            nxt = g.nodes[idx + 1] if idx + 1 < len(g.nodes) else None
            if nd.outputs[0] in outputs or (nxt is not None and nxt.outputs and nxt.outputs[0] in outputs):
                nodes.append(nd)  # the final projection stays replicated
                continue
            x, w = nd.inputs[0], consts[nd.inputs[1]]
            trans_b = int(nd.attrs.get("transB", 0)) if op == "Gemm" else 0
            groups = next((len(s.outputs) for s in g.nodes[idx + 1:idx + 3] if s.op_type == "Split"), 1)
            bias = nd.inputs[2] if len(nd.inputs) > 2 and nd.inputs[2] else None
            if x not in place:                       # column split
                nd.inputs[1] = new_const(w.name, shard_array(w.array, 0 if trans_b else 1, groups), w.data_type)
                if bias is not None:
                    b = consts[bias]
                    nd.inputs[2] = new_const(bias, shard_array(b.array, b.array.ndim - 1, groups), b.data_type)
                place[nd.outputs[0]] = last_axis(nd.outputs[0])
                nodes.append(nd)
            elif place[x] == last_axis(x):           # row split + all-reduce (+ bias once, after the reduction)
                nd.inputs[1] = new_const(w.name, shard_array(w.array, 1 if trans_b else 0), w.data_type)
                out = nd.outputs[0]
                partial = out + ":partial"
                nd.outputs[0] = partial
                nd.inputs = nd.inputs[:2]
                nodes.append(nd)
                reduced = out if bias is None else out + ":reduced"
                nodes.append(Node("ReduceSum", [partial], [reduced], nd.name + "/all_reduce", {"communicator": 0, "noop_with_empty_axes": 1}))
                if bias is not None:
                    nodes.append(Node("Add", [reduced, bias], [out], nd.name + "/bias"))
            else:
                raise NotImplementedError(f"{op} {nd.name}: activation sharded on axis {place[x]}, not the contraction axis")
            continue
        ins = [x for x in nd.inputs if x]
        sharded = [x for x in ins if x in place]
        if not sharded:
            nodes.append(nd)
            continue
        if op in unary_like:
            place[nd.outputs[0]] = place[nd.inputs[0]]
        elif op in OnnxStub._BINARY or op == "Where":
            acts = [x for x in ins if x not in consts]
            axes = {place.get(x) for x in acts}
            if len(axes) != 1:
                raise NotImplementedError(f"{op} {nd.name}: operands are placed differently ({axes})")
            ax = axes.pop()
            out_rank = len(shapes[nd.outputs[0]])
            for k, x in enumerate(nd.inputs):
                if x in consts:  # a broadcast constant that spans the sharded axis is split with it
                    c = consts[x]
                    cax = ax - (out_rank - c.array.ndim)
                    if cax >= 0 and c.array.shape[cax] == shapes[nd.outputs[0]][ax]:
                        nd.inputs[k] = new_const(x, shard_array(c.array, cax), c.data_type)
            place[nd.outputs[0]] = ax
        elif op == "RoPE":
            place[nd.outputs[0]] = place[nd.inputs[1]]
        elif op == "Transpose":
            perm = [int(p) for p in nd.attrs.get("perm") or range(len(shapes[nd.inputs[0]]))[::-1]]
            place[nd.outputs[0]] = perm.index(place[nd.inputs[0]])
        elif op == "Reshape":
            src, k = shapes[nd.inputs[0]], place[nd.inputs[0]]
            tgt = consts[nd.inputs[1]]
            dims = [int(v) for v in tgt.array]
            dims = [src[i] if v == 0 else v for i, v in enumerate(dims)]
            if -1 in dims:
                dims[dims.index(-1)] = int(np.prod(src)) // max(int(np.prod([v for v in dims if v != -1])), 1)
            left = int(np.prod(src[:k]))
            cand = [j for j in range(len(dims)) if int(np.prod(dims[:j])) == left and dims[j] % world == 0 and dims[j] >= world]
            if not cand:
                raise NotImplementedError(f"Reshape {nd.name}: no output axis lines up with sharded input axis {k} ({src} -> {dims})")
            j = cand[-1]
            dims[j] //= world
            nd.inputs[1] = new_const(tgt.name, np.array(dims, np.int64), I64)
            place[nd.outputs[0]] = j
        elif op == "Split":
            ax, k = int(nd.attrs.get("axis", 0)) % len(shapes[nd.inputs[0]]), place[nd.inputs[0]]
            if ax == k and len(nd.inputs) > 1 and nd.inputs[1] in consts:
                c = consts[nd.inputs[1]]
                nd.inputs[1] = new_const(c.name, c.array // world, c.data_type)
            for o in nd.outputs:
                place[o] = k
        elif op == "AttentionKVCache":
            if {place.get(x) for x in nd.inputs[2:5]} != {1}:
                raise NotImplementedError("AttentionKVCache: q, k, v must all be sharded by head (axis 1)")
            for cache in nd.inputs[:2]:
                if cache not in inputs:
                    raise NotImplementedError("AttentionKVCache: the caches must be graph inputs to be sharded by head")
                if cache not in place:
                    v = inputs[cache]
                    inputs[cache] = ValueInfo(v.name, v.elem_type, [d // world if i == 1 else d for i, d in enumerate(v.dims)])
                    place[cache] = 1
            for i in (6, 7):  # an FP8 cache's per-KV-head scales split with its heads
                if i >= len(nd.inputs) or place.get(nd.inputs[i]) == 0:
                    continue
                sc = nd.inputs[i]
                if sc in consts:
                    c = consts[sc]
                    nd.inputs[i] = new_const(c.name, shard_array(c.array, 0), c.data_type)
                    place[nd.inputs[i]] = 0
                elif sc in inputs:
                    v = inputs[sc]
                    inputs[sc] = ValueInfo(v.name, v.elem_type, [v.dims[0] // world])
                    place[sc] = 0
                else:
                    raise NotImplementedError("AttentionKVCache: k_scale / v_scale must be graph inputs or initializers")
            place[nd.outputs[0]] = 1
        elif op == "MatMul":
            a_ax, b_ax = place.get(nd.inputs[0]), place.get(nd.inputs[1])
            ra = len(shapes[nd.inputs[0]])
            if a_ax != b_ax or a_ax is None or a_ax >= ra - 2:
                raise NotImplementedError(f"MatMul {nd.name}: activation operands must be sharded on the same batch axis")
            place[nd.outputs[0]] = a_ax
        else:
            raise NotImplementedError(f"{op} {nd.name}: a sharded input reaches an operator with no tensor-parallel rule")
        nodes.append(nd)
    for o in g.outputs:
        if o.name in place:
            raise NotImplementedError(f"graph output {o.name} would be sharded on axis {place[o.name]}")
    used = {x for nd in nodes for x in nd.inputs}
    return Model(Graph(nodes, [t for n_, t in consts.items() if n_ in used], [inputs[v.name] for v in g.inputs], list(g.outputs),
                       f"{g.name}_{rank}"), m.ir_version, m.opset)
