"""`backend` -- Python mirror of the reference's pybind module `pyinfinitensor.backend`
(reference src/ffi/ffi_infinitensor.cc:441-638), bound over the C-ABI of include/it_b200.h with ctypes.

Same class / method names, argument order and error behaviour (RuntimeError on failure) as the
reference so that OnnxStub-style callers and the reference's Python tests read unchanged:

    rt = backend.CudaRuntime(0)
    h = backend.GraphHandler(rt)
    a = h.tensor([16, 4096], backend.DType.BFloat16); ...
    y = h.matmul(a, w, None, False, False, None, backend.ActType.Linear)
    h.data_malloc(); a.copyin_numpy(x); h.run(); out = y.copyout_numpy()

There is no CPU runtime here (`cpu_runtime()` raises): this package is the B200 kernel backend only.
"""
from __future__ import annotations

import ctypes
import os
import enum
from ctypes import POINTER, byref, c_char_p, c_double, c_int, c_int64, c_void_p

import numpy as np

from . import _lib as L

lib = L.lib


class DType(enum.IntEnum):  # ONNX enum, reference include/core/data_type.h:6-23
    Float32 = 1
    UInt8 = 2
    Int8 = 3
    UInt16 = 4
    Int16 = 5
    Int32 = 6
    Int64 = 7
    Bool = 9
    Float16 = 10
    Double = 11
    UInt32 = 12
    UInt64 = 13
    BFloat16 = 16


class ActType(enum.IntEnum):  # reference export_values: Linear/Relu/Sigmoid/Tanh
    Linear = 0
    Relu = 1
    Sigmoid = 2
    Tanh = 3


_NP = {1: np.float32, 2: np.uint8, 3: np.int8, 4: np.uint16, 5: np.int16, 6: np.int32, 7: np.int64, 9: np.bool_,
       10: np.float16, 11: np.float64, 12: np.uint32, 13: np.uint64, 16: np.uint16,  # bf16 travels as raw uint16
       17: np.uint8}  # FP8 E4M3 codes

_h = c_void_p
_sig = {
    "itb_runtime_create": (c_int, [c_int, c_int64, POINTER(_h)]),
    "itb_runtime_destroy": (c_int, [_h]),
    "itb_runtime_init_comm": (c_int, [_h, c_char_p, c_int, c_int]),
    "itb_runtime_init_comm_with_id": (c_int, [_h, c_void_p, c_int, c_int, c_int]),
    "itb_runtime_nccl_unique_id": (c_int, [c_void_p, c_int]),
    "itb_runtime_p2p_export": (c_int, [_h, c_void_p]),
    "itb_runtime_p2p_import": (c_int, [_h, c_void_p, c_int, c_int]),
    "itb_runtime_cuda_graph_cache_size": (c_int64, [_h]),
    "itb_runtime_cuda_graph_capture_count": (c_int64, [_h]),
    "itb_runtime_clear_cuda_graph_cache": (c_int, [_h]),
    "itb_runtime_kernel_launches": (c_int64, [_h]),
    "itb_runtime_stream": (c_void_p, [_h]),
    "itb_graph_create": (c_int, [_h, POINTER(_h)]),
    "itb_graph_destroy": (c_int, [_h]),
    "itb_graph_tensor": (c_int, [_h, POINTER(c_int), c_int, c_int, POINTER(c_int64)]),
    "itb_tensor_set_weight": (c_int, [_h, c_int64]),
    "itb_tensor_set_input": (c_int, [_h, c_int64]),
    "itb_tensor_set_output": (c_int, [_h, c_int64]),
    "itb_tensor_rank": (c_int, [_h, c_int64]),
    "itb_tensor_shape": (c_int, [_h, c_int64, POINTER(c_int)]),
    "itb_tensor_dtype": (c_int, [_h, c_int64]),
    "itb_tensor_bytes": (c_int64, [_h, c_int64]),
    "itb_tensor_device_ptr": (c_void_p, [_h, c_int64]),
    "itb_tensor_copyin": (c_int, [_h, c_int64, c_void_p, c_int64]),
    "itb_tensor_copyout": (c_int, [_h, c_int64, c_void_p, c_int64]),
    "itb_tensor_copyin_async": (c_int, [_h, c_int64, c_void_p, c_int64]),
    "itb_tensor_copyout_async": (c_int, [_h, c_int64, c_void_p, c_int64]),
    "itb_graph_add_op": (c_int, [_h, c_char_p, POINTER(c_int64), c_int, POINTER(c_int64), c_int, POINTER(c_int64),
                                 c_int, POINTER(c_double), c_int]),
    "itb_graph_num_ops": (c_int, [_h]),
    "itb_graph_op_type": (c_int, [_h, c_int, c_char_p, c_int]),
    "itb_graph_num_steps": (c_int, [_h]),
    "itb_graph_step": (c_int, [_h, c_int, c_char_p, c_int]),
    "itb_graph_topo_sort": (c_int, [_h]),
    "itb_graph_shape_infer": (c_int, [_h]),
    "itb_graph_optimize": (c_int, [_h]),
    "itb_graph_data_malloc": (c_int, [_h, c_int, c_int64]),
    "itb_graph_run": (c_int, [_h]),
    "itb_graph_run_without_sync": (c_int, [_h]),
    "itb_graph_run_with_cudagraph": (c_int, [_h]),
    "itb_graph_launch_cudagraph_async": (c_int, [_h]),
    "itb_graph_tune": (c_int, [_h]),
    "itb_graph_sync": (c_int, [_h]),
    "itb_graph_get_perf_time": (c_double, [_h]),
    "itb_perf_engine_save": (c_int, [c_char_p]),
    "itb_perf_engine_load": (c_int, [c_char_p]),
    "itb_perf_engine_size": (c_int64, []),
    "itb_perf_engine_clear": (None, []),
    "itb_graph_arena_bytes": (c_int64, [_h, c_int]),
}
for _n, (_r, _a) in _sig.items():
    _f = getattr(lib, _n)
    _f.restype, _f.argtypes = _r, _a

GRAPH_API_SYMBOLS = sorted(_sig)


def _ck(ret):
    if ret != 0:
        raise RuntimeError(L.last_error())  # pybind maps infini::Exception to RuntimeError


def cpu_runtime():
    raise RuntimeError("infinitensor_b200 is the B200 kernel backend: there is no CPU runtime and no CPU fallback")


class CudaRuntime:
    """reference CudaRuntimeObj (include/cuda/cuda_runtime.h:70-110) as bound at ffi_infinitensor.cc:449-456."""

    def __init__(self, device: int = 0, cuda_graph_cache_capacity: int = 16):
        self._h = _h()
        _ck(lib.itb_runtime_create(device, cuda_graph_cache_capacity, byref(self._h)))
        self.device = device

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.itb_runtime_destroy(h)

    @staticmethod
    def _preload_nccl():
        """Make sure the process holds ONE libnccl.so.2: the copy torch bundles (nvidia-nccl wheel) if present,
        so a later `import torch` finds its own symbols; the C side then picks up whatever is loaded."""
        import importlib.util
        import os
        try:
            spec = importlib.util.find_spec("nvidia.nccl")
            if spec and spec.submodule_search_locations:
                p = os.path.join(list(spec.submodule_search_locations)[0], "lib", "libnccl.so.2")
                if os.path.exists(p):
                    ctypes.CDLL(p, mode=ctypes.RTLD_GLOBAL)
        except Exception:
            pass

    def init_comm(self, name: str, world_size: int, rank: int):
        self._preload_nccl()
        _ck(lib.itb_runtime_init_comm(self._h, name.encode(), world_size, rank))

    def init_comm_with_id(self, unique_id: bytes, world_size: int, rank: int):
        self._preload_nccl()
        buf = ctypes.create_string_buffer(unique_id, len(unique_id))
        _ck(lib.itb_runtime_init_comm_with_id(self._h, buf, len(unique_id), world_size, rank))

    @staticmethod
    def nccl_unique_id() -> bytes:
        CudaRuntime._preload_nccl()
        buf = ctypes.create_string_buffer(256)
        n = lib.itb_runtime_nccl_unique_id(buf, 256)
        if n <= 0:
            raise RuntimeError(L.last_error())
        return buf.raw[:n]

    def p2p_export(self) -> bytes:
        """64-byte cudaIpc handle of this rank's NVLink comm workspace (for the fused one-shot all-reduce)."""
        buf = ctypes.create_string_buffer(64)
        _ck(lib.itb_runtime_p2p_export(self._h, buf))
        return buf.raw

    def p2p_import(self, handles, world_size: int, rank: int):
        """Map every rank's comm workspace; `handles` = list of the world's p2p_export() results in rank order."""
        blob = b"".join(handles)
        assert len(blob) == 64 * world_size
        buf = ctypes.create_string_buffer(blob, len(blob))
        _ck(lib.itb_runtime_p2p_import(self._h, buf, world_size, rank))

    def clear_cuda_graph_cache(self):
        _ck(lib.itb_runtime_clear_cuda_graph_cache(self._h))

    def cuda_graph_cache_size(self) -> int:
        return int(lib.itb_runtime_cuda_graph_cache_size(self._h))

    def cuda_graph_capture_count(self) -> int:
        return int(lib.itb_runtime_cuda_graph_capture_count(self._h))

    def kernel_launches(self) -> int:
        return int(lib.itb_runtime_kernel_launches(self._h))

    def stream(self) -> int:
        return int(lib.itb_runtime_stream(self._h) or 0)


class HostPlanRuntime(CudaRuntime):
    """Planning-only runtime (device -1): build / shape-infer / memory-plan graphs without a GPU.
    Nothing executes on it -- run() raises.  Used by the CPU test tier, never as a fallback."""

    def __init__(self):
        self._h = _h()
        _ck(lib.itb_runtime_create(-1, 0, byref(self._h)))
        self.device = -1


class Tensor:
    """reference TensorObj bindings (ffi_infinitensor.cc:478-540)."""

    def __init__(self, handler: "GraphHandler", tid: int):
        self._g, self._id = handler, int(tid)

    def _gh(self):
        return self._g._h

    def fuid(self) -> int:
        return self._id

    def shape(self):
        r = lib.itb_tensor_rank(self._gh(), self._id)
        if r < 0:
            raise RuntimeError(L.last_error())
        d = (c_int * max(r, 1))()
        _ck(lib.itb_tensor_shape(self._gh(), self._id, d))
        return [int(d[i]) for i in range(r)]

    def dtype(self) -> int:
        return int(lib.itb_tensor_dtype(self._gh(), self._id))

    def nbytes(self) -> int:
        return int(lib.itb_tensor_bytes(self._gh(), self._id))

    def device_ptr(self) -> int:
        return int(lib.itb_tensor_device_ptr(self._gh(), self._id) or 0)

    def set_weight(self):
        _ck(lib.itb_tensor_set_weight(self._gh(), self._id))

    def set_input(self):
        _ck(lib.itb_tensor_set_input(self._gh(), self._id))

    def set_output(self):
        _ck(lib.itb_tensor_set_output(self._gh(), self._id))

    # -- host <-> device (HOST buffers; synchronous like the reference's cudaMemcpy, cuda_runtime.cc:162-166)
    def copyin_numpy(self, arr: np.ndarray):
        arr = np.ascontiguousarray(arr)
        want = _NP[self.dtype()]
        if arr.dtype.itemsize != np.dtype(want).itemsize:
            raise RuntimeError(f"copyin_numpy: itemsize {arr.dtype.itemsize} != tensor itemsize {np.dtype(want).itemsize}")
        if list(arr.shape) != self.shape():
            raise RuntimeError(f"copyin_numpy: shape {list(arr.shape)} != tensor shape {self.shape()}")
        _ck(lib.itb_tensor_copyin(self._gh(), self._id, arr.ctypes.data_as(c_void_p), arr.nbytes))

    def copyout_numpy(self) -> np.ndarray:
        out = np.empty(self.shape(), dtype=_NP[self.dtype()])
        _ck(lib.itb_tensor_copyout(self._gh(), self._id, out.ctypes.data_as(c_void_p), out.nbytes))
        return out

    def _copyin_list(self, vals, npdt):
        a = np.asarray(vals, dtype=npdt).reshape(self.shape())
        self.copyin_numpy(a)

    def copyin_float(self, v): self._copyin_list(v, np.float32)
    def copyin_int32(self, v): self._copyin_list(v, np.int32)
    def copyin_int64(self, v): self._copyin_list(v, np.int64)
    def copyin_int8(self, v): self._copyin_list(v, np.int8)
    def copyin_uint8(self, v): self._copyin_list(v, np.uint8)
    def copyin_float16(self, v): self._copyin_list(v, np.uint16)
    def copyout_float(self): return self.copyout_numpy().ravel().tolist()
    def copyout_int32(self): return self.copyout_numpy().ravel().tolist()
    def copyout_int64(self): return self.copyout_numpy().ravel().tolist()
    def copyout_int8(self): return self.copyout_numpy().ravel().tolist()
    def copyout_uint8(self): return self.copyout_numpy().ravel().tolist()
    def copyout_float16(self): return self.copyout_numpy().view(np.uint16).ravel().tolist()

    # -- stream-ordered variants for the serving loop (pinned host memory; pair with handler.sync())
    def copyin_async(self, host_ptr: int, nbytes: int):
        _ck(lib.itb_tensor_copyin_async(self._gh(), self._id, c_void_p(host_ptr), nbytes))

    def copyout_async(self, host_ptr: int, nbytes: int):
        _ck(lib.itb_tensor_copyout_async(self._gh(), self._id, c_void_p(host_ptr), nbytes))


class PerfEngine:
    """The process-wide PerfEngine table that `GraphHandler.tune()` fills (reference include/core/perf_engine.h:8-50)."""

    @staticmethod
    def save(path: str): _ck(lib.itb_perf_engine_save(os.fsencode(path)))

    @staticmethod
    def load(path: str): _ck(lib.itb_perf_engine_load(os.fsencode(path)))

    @staticmethod
    def size() -> int: return int(lib.itb_perf_engine_size())

    @staticmethod
    def clear(): lib.itb_perf_engine_clear()


def _ids(ts):
    return [(-1 if t is None else t._id) for t in ts]


class GraphHandler:
    """reference GraphHandlerObj (include/core/graph_handler.h:15-159) as bound at ffi_infinitensor.cc:548-638."""

    head_widths = (64, 128)  # decode attention / RoPE head widths (64: extension; the reference's are 128)
    rope_inv_freq = True  # RoPE takes the model's frequencies as an optional inv_freq input (extension)
    sliding_window = True  # AttentionKVCache takes a sliding window (extension)
    rolling_cache = True  # a windowed AttentionKVCache's caches may be a ring (extension)

    def __init__(self, runtime: CudaRuntime):
        if not isinstance(runtime, CudaRuntime):
            raise RuntimeError("GraphHandler needs a backend.CudaRuntime")
        self._rt = runtime
        self._h = _h()
        _ck(lib.itb_graph_create(runtime._h, byref(self._h)))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.itb_graph_destroy(h)

    # ---- tensors / generic op insertion
    def tensor(self, dims, dtype: int) -> Tensor:
        d = (c_int * max(len(dims), 1))(*[int(x) for x in dims])
        tid = c_int64(-1)
        _ck(lib.itb_graph_tensor(self._h, d, len(dims), int(dtype), byref(tid)))
        return Tensor(self, tid.value)

    def _op(self, name, inputs, outputs, iattrs=(), fattrs=()):
        ins = _ids(inputs)
        outs = _ids(outputs)
        ia = [int(x) for x in iattrs]
        fa = [float(x) for x in fattrs]
        cin = (c_int64 * max(len(ins), 1))(*ins)
        cout = (c_int64 * max(len(outs), 1))(*outs)
        cia = (c_int64 * max(len(ia), 1))(*ia)
        cfa = (c_double * max(len(fa), 1))(*fa)
        _ck(lib.itb_graph_add_op(self._h, name.encode(), cin, len(ins), cout, len(outs), cia, len(ia), cfa, len(fa)))
        res = [Tensor(self, cout[i]) for i in range(len(outs))]
        return res

    def _op1(self, name, inputs, output, iattrs=(), fattrs=()):
        return self._op(name, inputs, [output], iattrs, fattrs)[0]

    # ---- operators (same names / argument order as the reference handler)
    def conv(self, input, weight, output, ph, pw, sh, sw, dh, dw):
        return self._op1("Conv", [input, weight], output, [ph, pw, sh, sw, dh, dw])

    def matmul(self, a, b, y, transA, transB, bias, act, matmul_compute_type="default", w_scale=None):
        """w_scale (extension, SURVEY 8(f-4)): `b` holds FP8 E4M3 codes (dtype 17) [K, N] and w_scale is its f32 per-column scale;
        the product is X . (codes * scale), dequantised inside the GEMM."""
        ins = [a, b] + ([bias] if bias is not None else []) + ([w_scale] if w_scale is not None else [])
        return self._op1("MatMul", ins, y, [int(transA), int(transB), int(act), 1 if w_scale is not None else 0])

    def matMulNBits(self, a, b, scales, zero_points, y, K, N, block_size, bits=4, g_idx=None, bias=None):
        """com.microsoft MatMulNBits (extension), 4-bit weights with block-wise scales: y[.., N] = a[.., K] . W,
        W[k, n] = (q[n, k] - z[n, k // block_size]) * scales[n * (K // block_size) + k // block_size].  b: uint8 [N, K // bs, bs // 2]
        (even k in the low nibble); zero_points: None (z = 8) or uint8 nibble-packed [N * (K // bs) // 2].  a / scales / y: f16 or bf16.
        g_idx and bias are the operator's optional inputs; the backend refuses them."""
        opt = [zero_points, g_idx, bias]
        ins = [a, b, scales] + [t for t in opt if t is not None]
        return self._op1("MatMulNBits", ins, y, [int(K), int(N), int(bits), int(block_size)] + [int(t is not None) for t in opt])

    def batchNormalization(self, input, output, mean, var, scale, bias, momentum, eps, training):
        return self._op1("BatchNormalization", [input, mean, var, scale, bias], output, [int(training)], [momentum, eps])

    def layerNormalization(self, input, scale, output, bias, eps, axis, stash_type):
        return self._op1("LayerNormalization", [input, scale] + ([bias] if bias is not None else []), output,
                         [axis, stash_type], [eps])

    def RMSNorm(self, input, weight, output):
        return self._op1("RMSNorm", [input, weight], output)

    def maxPool(self, input, output, kh, kw, dh, dw, ph, pw, sh, sw, ceilMode):
        return self._op1("MaxPool", [input], output, [kh, kw, dh, dw, ph, pw, sh, sw, ceilMode])

    def avgPool(self, input, output, kh, kw, dh, dw, ph, pw, sh, sw, ceilMode):
        return self._op1("AveragePool", [input], output, [kh, kw, dh, dw, ph, pw, sh, sw, ceilMode])

    def _bin(name):
        def f(self, a, b, c):
            return self._op1(name, [a, b], c)
        return f

    add, sub, mul, div, pow = _bin("Add"), _bin("Sub"), _bin("Mul"), _bin("Div"), _bin("Pow")
    min, max = _bin("Min"), _bin("Max")
    less, equal, greater = _bin("Less"), _bin("Equal"), _bin("Greater")

    def _un(name):
        def f(self, x, y):
            return self._op1(name, [x], y)
        return f

    relu, silu, gelu, sigmoid, tanh = _un("Relu"), _un("Silu"), _un("Gelu"), _un("Sigmoid"), _un("Tanh")
    hardSigmoid, hardSwish, erf, abs, sqrt, neg = (_un("HardSigmoid"), _un("HardSwish"), _un("Erf"), _un("Abs"),
                                                   _un("Sqrt"), _un("Neg"))
    exp, identity = _un("Exp"), _un("Identity")
    del _bin, _un

    def softmax(self, x, y, axis):
        return self._op1("Softmax", [x], y, [axis])

    def flatten(self, s, y, axis):
        return self._op1("Flatten", [s], y, [axis])

    def transpose(self, data, transposed, perm):
        return self._op1("Transpose", [data], transposed, list(perm))

    def reshape(self, data, reshaped, shape):
        return self._op1("Reshape", [data], reshaped, list(shape))

    def squeeze(self, input, output, axes):
        return self._op1("Squeeze", [input], output, list(axes))

    def unsqueeze(self, input, output, axes):
        return self._op1("Unsqueeze", [input], output, list(axes))

    def leakyRelu(self, input, output, alpha):
        return self._op1("LeakyRelu", [input], output, [], [float(alpha)])

    def elu(self, input, output, alpha):
        return self._op1("Elu", [input], output, [], [float(alpha)])

    def depthToSpace(self, input, output, blocksize, mode):
        if isinstance(mode, bytes):
            mode = mode.decode()
        return self._op1("DepthToSpace", [input], output, [int(blocksize), 1 if mode == "CRD" else 0])

    def concat(self, inputs, output, dim):
        return self._op1("Concat", list(inputs), output, [dim])

    def attentionKVCache(self, input_k_cache, input_v_cache, input_q, input_k, input_v, position_id, output_matmul,
                         per_row_positions=False, k_scale=None, v_scale=None, window=0, rolling=False):
        """per_row_positions (extension, SURVEY 8(f-3)): batch row b attends up to / appends at position_id[b]; the default is
        the reference's rule -- element 0 for every row (attention_kvcache.cu:17).
        k_scale / v_scale (extension): the caches hold FP8 E4M3 codes (dtype 17), element value e4m3(code) * scale[KV head];
        both f32 [Hkv], given together, exactly when the caches are FP8.  One token per step, f16 / bf16 q / k / v.
        window (extension): sliding-window attention, the query at position P attends over cache rows (P - window, P] only
        (HF's sliding_window); 0 = no window.  Decode and prompt steps, every cache type; a negative window is refused.
        rolling (extension, needs a window): the caches [B, Hkv, S_max, D] are a ring, position P in row P mod S_max, so S_max
        bounds the window rather than the context (Mistral's rolling buffer cache).  S_max >= window, S_max % 64 == 0, and a
        prompt chunk of S tokens needs S_max >= window + S - 1."""
        ins = [input_k_cache, input_v_cache, input_q, input_k, input_v, position_id]
        if (k_scale is None) != (v_scale is None):
            raise ValueError("attentionKVCache: k_scale and v_scale go together")
        if k_scale is not None:
            ins += [k_scale, v_scale]
        attrs = [int(bool(per_row_positions)), int(window)] if window else ([1] if per_row_positions else [])
        if rolling:
            attrs = [int(bool(per_row_positions)), int(window), 1]
        return self._op1("AttentionKVCache", ins, output_matmul, attrs)

    def RoPE(self, pos, input, output, dim_head=128, inv_freq=None):
        """dim_head (extension): rotate-half within heads of this width; the reference fixes it at 128 (rope.cc:25).
        inv_freq (extension): an f32 [dim_head / 2] tensor of the model's frequencies (HF's `inv_freq` buffer, e.g.
        `graphs.rope_inv_freq`); column pair c rotates by fp32(p * inv_freq[c]) instead of p * 10000^(-2c / dim_head)."""
        ins = [pos, input] + ([inv_freq] if inv_freq is not None else [])
        return self._op1("RoPE", ins, output, [] if dim_head == 128 else [int(dim_head)])

    def split(self, input, outputs, axis, numOrRatio):
        if isinstance(numOrRatio, int):
            n, ia = numOrRatio, [axis, numOrRatio]
        else:
            n, ia = len(numOrRatio), [axis, -1] + list(numOrRatio)
        outs = list(outputs) if outputs is not None else [None] * n
        return self._op("Split", [input], outs, ia)

    def gather(self, data, indices, output, axis):
        return self._op1("Gather", [data, indices], output, [axis])

    def reduceMean(self, data, reduced, axes, keepdims):
        return self._op1("ReduceMean", [data], reduced, [int(keepdims)] + (list(axes) if axes is not None else []))

    def reduceSum(self, data, reduced, axes, keepdims):
        return self._op1("ReduceSum", [data], reduced, [int(keepdims)] + (list(axes) if axes is not None else []))

    def slice(self, input, output, starts, ends, axes, steps):
        n = len(starts)
        ia = [n] + list(starts) + list(ends)
        ia += [1] + list(axes) if axes is not None else [0]
        ia += [1] + list(steps) if steps is not None else [0]
        return self._op1("Slice", [input], output, ia)

    def pad(self, input, output, pads, axes):
        ia = [len(pads)] + list(pads)
        ia += [1] + list(axes) if axes is not None else [0]
        return self._op1("Pad", [input], output, ia)

    def cast(self, input, output, to):
        return self._op1("Cast", [input], output, [int(to)])

    def expand(self, input, output, dims):
        return self._op1("Expand", [input], output, list(dims))

    def where(self, inputX, inputY, condition, output):
        return self._op1("Where", [inputX, inputY, condition], output)

    def allReduceSum(self, input, output): return self._op1("AllReduceSum", [input], output)
    def allReduceProd(self, input, output): return self._op1("AllReduceProd", [input], output)
    def allReduceMin(self, input, output): return self._op1("AllReduceMin", [input], output)
    def allReduceMax(self, input, output): return self._op1("AllReduceMax", [input], output)
    def allReduceAvg(self, input, output): return self._op1("AllReduceAvg", [input], output)

    def allGather(self, input, outputs, n):
        outs = list(outputs) if outputs is not None else [None] * n
        return self._op("AllGather", [input], outs, [n])

    def getDims(self, x):
        return x.shape()

    # ---- modifiers / runtime
    def topo_sort(self):
        return lib.itb_graph_topo_sort(self._h) == 0

    def optimize(self):
        _ck(lib.itb_graph_optimize(self._h))

    def shape_infer(self):
        _ck(lib.itb_graph_shape_infer(self._h))

    def operators(self):
        buf = ctypes.create_string_buffer(64)
        out = []
        for i in range(lib.itb_graph_num_ops(self._h)):
            _ck(lib.itb_graph_op_type(self._h, i, buf, 64))
            out.append(buf.value.decode())
        return out

    def schedule(self):
        """The fused execution schedule: one "Kind:Op[+Op...]" string per step."""
        buf = ctypes.create_string_buffer(256)
        out = []
        n = lib.itb_graph_num_steps(self._h)
        if n < 0:
            raise RuntimeError(L.last_error())
        for i in range(n):
            _ck(lib.itb_graph_step(self._h, i, buf, 256))
            out.append(buf.value.decode())
        return out

    def data_malloc(self, useNaiveAllocator: bool = False, memPoolSize: int = 0):
        _ck(lib.itb_graph_data_malloc(self._h, int(useNaiveAllocator), int(memPoolSize)))

    def tune(self):
        _ck(lib.itb_graph_tune(self._h))

    def run(self):
        _ck(lib.itb_graph_run(self._h))

    def run_without_sync(self):
        _ck(lib.itb_graph_run_without_sync(self._h))

    def run_with_cudagraph(self):
        _ck(lib.itb_graph_run_with_cudagraph(self._h))

    def launch_cudagraph_async(self):
        _ck(lib.itb_graph_launch_cudagraph_async(self._h))

    def sync(self):
        _ck(lib.itb_graph_sync(self._h))

    def get_perf_time(self) -> float:
        return float(lib.itb_graph_get_perf_time(self._h))

    def arena_bytes(self):
        return int(lib.itb_graph_arena_bytes(self._h, 0)), int(lib.itb_graph_arena_bytes(self._h, 1))
