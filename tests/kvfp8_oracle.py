"""Oracle for AttentionKVCache over an FP8 E4M3 KV cache (the kernels' extension; the reference has no FP8 cache).

Semantics (include/it_b200.h, it_b200_attention_kvcache_fp8): a cache element is e4m3(code) * scale[KV head]; the step
quantises the new row p as code = RN-even-satfinite(fp32(x) / scale[h]) with the division correctly rounded, then attends
over rows 0 .. p read back from their codes:  s_j = (q . e4m3(code_k,j)) * scale_k[h] / sqrt(D),  softmax,
out = (sum_j w_j e4m3(code_v,j)) * scale_v[h], rounded to the activation type once.

`quantise` restates the quantiser bit for bit (numpy's float32 division is IEEE, correctly rounded); `attention` is the float64
reference with a per-element bound, `emulate32` follows the kernels' fp32 order of operations, so that the bound can be shown
to hold for it and to catch arithmetic slips.  The graph oracle (tests/llama_oracle.py) runs `append` and `attention` for
FP8 caches."""
import math

import numpy as np

import oracle as O

F32, F16, BF16 = 1, 10, 16
E4M3_MAX = 448.0


def _table() -> np.ndarray:
    t = np.zeros(256, np.float64)
    for c in range(256):
        e, m = (c >> 3) & 15, c & 7
        if e == 15 and m == 7:
            t[c] = np.nan
            continue
        v = (m / 8.0) * 2.0 ** -6 if e == 0 else (1.0 + m / 8.0) * 2.0 ** (e - 7)
        t[c] = -v if c & 0x80 else v
    return t


DECODE = _table()  # code -> value (float64; codes 0x7F / 0xFF are NaN)


def decode(codes) -> np.ndarray:
    return DECODE[np.asarray(codes, np.uint8)]


def e4m3(x) -> np.ndarray:
    """float32 -> E4M3 codes: round to nearest, ties to even, saturated to +-448; NaN -> 0x7F (sign kept)."""
    x = np.asarray(x, np.float32)
    mag = np.abs(x).astype(np.float64)
    pos = DECODE[:127]  # the 127 finite non-negative values, ascending
    m = np.minimum(np.nan_to_num(mag, nan=0.0), E4M3_MAX)
    hi = np.clip(np.searchsorted(pos, m, side="left"), 0, 126)
    lo = np.clip(hi - 1, 0, 126)
    dlo, dhi = m - pos[lo], pos[hi] - m
    code = np.where((dhi < dlo) | ((dhi == dlo) & (hi % 2 == 0)), hi, lo).astype(np.uint8)
    code = np.where(np.isnan(mag), np.uint8(0x7F), code)
    return np.where(np.signbit(x), code | 0x80, code).astype(np.uint8)


def quantise(x, scale) -> np.ndarray:
    """The append's quantiser: e4m3(fp32(x) / scale), the fp32 division correctly rounded.  scale broadcasts against x."""
    return e4m3(np.asarray(x, np.float32) / np.asarray(scale, np.float32))


def quantise_reciprocal(x, scale) -> np.ndarray:
    """A quantiser that multiplies by fp32(1 / scale) -- not the kernels' rule; the tests show it differs."""
    return e4m3(np.asarray(x, np.float32) * (np.float32(1) / np.asarray(scale, np.float32)))


def fill(values, axis_heads=1):
    """Quantise float values [B, H, S, D] for an FP8 cache: scale[h] = amax of head h / 448 (the rule graphs.py applies)."""
    v = np.asarray(values, np.float32)
    red = tuple(i for i in range(v.ndim) if i != axis_heads)
    scale = (np.maximum(np.abs(v).max(axis=red), 1e-12).astype(np.float32) / np.float32(E4M3_MAX)).astype(np.float32)
    shp = [1] * v.ndim
    shp[axis_heads] = -1
    return quantise(v, scale.reshape(shp)), scale


def append(kc, vc, k, v, ksc, vsc, pos):
    """In place on the code caches kc / vc [B, Hkv, S, D] uint8: row pos[b] of every KV head <- quantise(k / v).
    k / v [B, Hkv, 1, D] (float32 values of the activation type, RoPE already applied to k)."""
    B, Hkv = kc.shape[:2]
    for b in range(B):
        p = int(pos[b])
        kc[b, :, p] = quantise(k[b, :, 0], ksc[:, None])
        vc[b, :, p] = quantise(v[b, :, 0], vsc[:, None])


def _ulp(x, dt):
    mant = {F16: 10, BF16: 7, F32: 23}[dt]
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -126)))
    if dt == F16:
        e = np.maximum(e, -14)
    return 2.0 ** (e - mant)


def attention(kc, vc, ksc, vsc, q, pos, dt):
    """Float64 reference over the dequantised caches (after the append) and its per-element bound.
    q [B, Hq, 1, D] float values; pos one per batch row.  Returns (ref [B, Hq, 1, D] float64, bound same shape):
        |got - ref| <= ulp_T(|ref|) + 2^-15 sum_j w_j |v_j| + 64 2^-24 sum_j w_j a_j |v_j - ref|,  a_j = sum_i |q_i k_ji|
    scaled like s_j: the output rounded to T once (an ulp allows a rounding across a binade), the fp32 softmax / P.V / merge
    chains (with the hi + lo split of P in the grouped-query kernel), and an fp32 error of up to 64 units in every score."""
    B, Hkv, S, D = kc.shape
    Hq = q.shape[1]
    G = Hq // Hkv
    ref = np.zeros((B, Hq, 1, D))
    bound = np.zeros((B, Hq, 1, D))
    for b in range(B):
        p = int(pos[b])
        K = decode(kc[b, :, :p + 1]) * np.asarray(ksc, np.float64)[:, None, None]
        V = decode(vc[b, :, :p + 1]) * np.asarray(vsc, np.float64)[:, None, None]
        Q = np.asarray(q[b, :, 0], np.float64).reshape(Hkv, G, D)
        s = np.einsum("hgd,hsd->hgs", Q, K) / math.sqrt(D)
        a = np.einsum("hgd,hsd->hgs", np.abs(Q), np.abs(K)) / math.sqrt(D)
        w = np.exp(s - s.max(-1, keepdims=True))
        w /= w.sum(-1, keepdims=True)
        r = np.einsum("hgs,hsd->hgd", w, V)
        dev = np.abs(V[:, None, :, :] - r[:, :, None, :])
        t2 = np.einsum("hgs,hsd->hgd", w, np.abs(V))
        t3 = np.einsum("hgs,hgsd->hgd", w * a, dev)
        ref[b, :, 0] = r.reshape(Hq, D)
        bound[b, :, 0] = (2.0 ** -15 * t2 + 64 * 2.0 ** -24 * t3).reshape(Hq, D)
    return ref, bound + _ulp(ref, dt)


def violations(got, ref, bound):
    return np.argwhere(~(np.abs(np.asarray(got, np.float64) - ref) <= bound))


def emulate32(kc, vc, ksc, vsc, q, k, v, pos, rows_per_chunk=128, bugs=()):
    """Float32 emulation of attn_stream_kv8_kernel's arithmetic (G = 1) for one batch row set, appending in place.
    Chunks of `rows_per_chunk` cache rows are folded with a running (m, l, acc) as the kernel does, the appended row last.
    `bugs` injects slips the bound must catch: 'scale_twice', 'neighbour_scale', 'unquantised_append', 'reciprocal',
    'chunk_off_by_one'."""
    f = np.float32
    B, H, S, D = kc.shape
    out = np.zeros((B, H, 1, D), np.float32)
    for b in range(B):
        p = int(pos[b])
        for h in range(H):
            hs = (h + 1) % H if "neighbour_scale" in bugs else h
            quant = quantise_reciprocal if "reciprocal" in bugs else quantise
            kcode = quant(k[b, h, 0], ksc[h])
            vcode = quant(v[b, h, 0], vsc[h])
            kc[b, h, p] = kcode
            vc[b, h, p] = vcode
            qs = f(ksc[hs]) * f(1.0 / math.sqrt(D))
            if "scale_twice" in bugs:
                qs = f(qs * f(ksc[hs]))
            qf = (np.asarray(q[b, h, 0], np.float32) * qs).astype(np.float32)
            last = p - 1 if "chunk_off_by_one" in bugs else p  # the slip drops the last cache row before the append
            m, l, acc = f(-np.inf), f(0), np.zeros(D, np.float32)
            for c0 in range(0, max(last, 0), rows_per_chunk):
                c1 = min(c0 + rows_per_chunk, last)
                K = decode(kc[b, h, c0:c1]).astype(np.float32)
                V = decode(vc[b, h, c0:c1]).astype(np.float32)
                s = (K @ qf).astype(np.float32)
                mx = f(max(m, s.max()))
                corr = f(np.exp(f(m - mx))) if m > -np.inf else f(0)
                pw = np.exp((s - mx).astype(np.float32)).astype(np.float32)
                l = f(l * corr + pw.sum(dtype=np.float32))
                acc = (acc * corr + pw @ V).astype(np.float32)
                m = mx
            if "unquantised_append" in bugs:
                kn, vn = np.asarray(k[b, h, 0], np.float32), np.asarray(v[b, h, 0], np.float32) / f(vsc[hs])
                kn = kn / f(ksc[h])
            else:
                kn, vn = decode(kcode).astype(np.float32), decode(vcode).astype(np.float32)
            d = f(kn @ qf)
            mx = f(max(m, d))
            corr = f(np.exp(f(m - mx))) if m > -np.inf else f(0)
            pn = f(np.exp(f(d - mx)))
            l = f(l * corr + pn)
            acc = (acc * corr + pn * vn).astype(np.float32)
            out[b, h, 0] = acc / l * f(vsc[hs])
    return out

