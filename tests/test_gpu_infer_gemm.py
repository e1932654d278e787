"""The batch-inference kernels (deep-prove_b200/csrc/infer.cu) against a plain integer reference, layer by layer, at tile edges
and value extremes, driven through dp_infer_plan / dp_infer_run directly.

k_infer_gemm<MODE> is an mma.sync m16n8k32 s8 x s8 -> s32 GEMM on 64 x 64 block tiles (M = GEMM rows, N = outputs, K = the
reduction, zero-padded to Kp, a multiple of 32).  Each case group reaches these cells:
  DENSE_CASES    MODE 0 (Dense): N in {1, 7, 8, 63, 64, 65, 129} (ragged N tiles, the n >= N guard), K in {1, 3, 31, 32, 33,
                 100, 1024} (the zero-padded Kp tail, up to 32 k-steps), batches of {1, 63, 64, 65, 129} inputs (ragged M tiles)
  MATMUL_CASES   MODE 1 (MatMul, K % 4 != 0: K in {1, 2, 3, 5}, byte loads) and MODE 0 (K in {36, 64}; K = 36 reads past each
                 row's end into the next row), R in {1, 3, 17} (R = 3 and 17: an input's rows straddle M tiles), C in {1, 5, 64, 70},
                 the right matrix stored [K][C] or [C][K], with and without bias; the "bufend" cases end the last input's last row
                 at the end of the device buffer, so the tail read lands in its slack
  CONV_CASES     MODE 2 (the implicit-GEMM gather): nw in {4, 8, 16, 32} (nw = 4: P = 16 positions, four inputs per M tile),
                 kx in {1, 3, 4}, rn in {1, 3, 5}, kw in {1, 3, 70}, kept outputs u0 < kw and u1 != u2 (the epilogue's mask),
                 taps that are zero for every output channel (pruned from K) and an all-zero filter (K = 0: bias on kept positions)
  every group    inputs and weights at random int8, pinned at -128 / 127, and one-hot inputs; each case stores int32 (GEMM alone),
                 int8 (fused Requant) or int8 through the fused Requant + Relu
  EDGE           the exactness bound 128 * sum|w| + |b| = 2^31 - 1 reached exactly by a 2^17 - 1 long row (4096 k-steps), and
                 refused one past it
  STACKS         the unfused element-wise kernels (k_infer_requant / _relu / _pool on int8 and int32 tensors), Requant clamps at
                 both ends and rounding ties, and how many launches each stack takes (what the plan fuses)
  ERROR_CASES    per-input error bits 1, 2 (fused Requant), 4, 8 (unfused Relu / Maxpool on int32) and 16 (an input outside the
                 8-bit domain) with failing inputs interleaved among passing ones in shared M tiles (MatMul R = 3, Conv P = 16)
  REFUSALS       every dp_infer_plan refusal, each naming its node

The reference (`ref_forward`) restates each node in numpy integers; test_reference_equals_checker pins it to the CPU checker's
inference (oracle_model_io.model_output) on power-of-two stacks, which is what lets the GPU tests compare against it at shapes
the checker does not take.  Every output word of every input and every input's error bits are compared; a mismatch names the
first input and element that differ.
"""
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import zlib

import numpy as np
import pytest
from scipy import signal

import models
import oracle_model_io as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DENSE, REQUANT, RELU, CONV, POOL, MATMUL = models.DENSE, models.REQUANT, models.RELU, models.CONV, models.POOL, models.MATMUL
I32_MAX = (1 << 31) - 1


class InferNode(C.Structure):
    """dp_infer_node (include/deepprove_b200.h)"""
    _fields_ = [("kind", C.c_uint32), ("dims", C.c_uint32 * 7), ("shift", C.c_uint32), ("clamp_size", C.c_uint32),
                ("intermediate_bits", C.c_uint32), ("multiplier", C.c_int64), ("weights", C.c_void_p), ("bias", C.c_void_p)]


class Node:
    """one dp_infer_node with its weights as int64 arrays"""
    def __init__(self, kind, dims=(), weights=None, bias=None, shift=0, clamp_size=0, intermediate_bits=0, multiplier=0):
        self.kind, self.dims = kind, tuple(int(d) for d in dims)
        self.weights = None if weights is None else np.ascontiguousarray(weights, dtype=np.int64).reshape(-1)
        self.bias = None if bias is None else np.ascontiguousarray(bias, dtype=np.int64).reshape(-1)
        self.shift, self.clamp_size, self.intermediate_bits, self.multiplier = shift, clamp_size, intermediate_bits, multiplier


def dense(w, b=None):
    w = np.asarray(w)
    return Node(DENSE, w.shape, w, b)


def matmul(R, K, Cc, stored, transposed, b=None):
    """stored: [K][C], or [C][K] when transposed"""
    return Node(MATMUL, (R, K, Cc, int(transposed)), stored, b)


def conv(filt, b, nw, unpadded):
    kw, kx, rn, _ = np.asarray(filt).shape
    return Node(CONV, (kw, kx, nw, rn) + tuple(unpadded), filt, b)


def requant(shift, clamp_size, intermediate_bits, multiplier):
    return Node(REQUANT, shift=shift, clamp_size=clamp_size, intermediate_bits=intermediate_bits, multiplier=multiplier)


def relu():
    return Node(RELU)


def pool(c, h, w):
    return Node(POOL, (c, h, w))


def nodes_from_desc(desc, data):
    """layer descriptors (models.py, read as dph_model_context_new reads them) -> the dp_infer_node list the host builds"""
    out, k = [], 0
    data = np.asarray(data, dtype=np.int64)

    def take(n):
        nonlocal k
        k += n
        return data[k - n: k]
    for d in np.asarray(desc, dtype=np.int64).reshape(-1, 9).tolist():
        kind = d[0]
        if kind == DENSE:
            w = take(d[1] * d[2]).reshape(d[1], d[2])
            out.append(dense(w, take(d[1])))
        elif kind == REQUANT:               # {right_shift, fp_scale, multiplier, intermediate_bits}
            shift = d[1] + d[2]
            out.append(requant(shift, d[4] + (d[3] - 1).bit_length() - shift, d[4], d[3]))
        elif kind == RELU:
            out.append(relu())
        elif kind == CONV:                  # {kw, kx, nw, real_nw, unpadded_out[3]}
            filt = take(d[1] * d[2] * d[4] * d[4]).reshape(d[1], d[2], d[4], d[4])
            out.append(conv(filt, take(d[1]), d[3], d[5:8]))
        elif kind == POOL:
            out.append(pool(*d[1:4]))
        elif kind == MATMUL:                # {R, K, C, transposed, has_bias}
            w = take(d[2] * d[3])
            out.append(matmul(d[1], d[2], d[3], w, d[4], take(d[3]) if d[5] else None))
    return out


# ---- reference: each node in numpy integers ---------------------------------------------------------------------------
def _any(mask):
    return mask.reshape(mask.shape[0], -1).any(axis=1)


def ref_requant(v, nd):
    """tmp = v m + 2^(shift-1), cl = tmp >> shift, out = clip(cl, -127, 127); bit 1 when |v| > 2^intermediate_bits, bit 2 when cl lies
    outside [-2^(size-1), 2^(size-1)).  In Python integers: v m may not fit int64."""
    lim, half = 1 << nd.intermediate_bits, 1 << (nd.clamp_size - 1)
    cl = (v.astype(object) * int(nd.multiplier) + (1 << (nd.shift - 1))) >> nd.shift
    err = np.where(_any((v > lim) | (v < -lim)), 1, 0) | np.where(_any((cl < -half) | (cl >= half)), 2, 0)
    return np.minimum(np.maximum(cl, -127), 127).astype(np.int64), err, cl


def ref_conv(x, nd):
    """the FFT convolution's flat-index rule (oracle/conv.hpp fft_conv: the input row reversed, the filter placed by index_w in the
    top-left of an nw x nw grid, the product read back through index_u): output channel o at position p = i nw + j is
    sum_{c,a,b} w[o][c][a][b] x[c][p + a nw + b], a term being 0 when p + a nw + b >= nw^2; then + bias, then 0 unless o < u0,
    i < u1 and j < u2 (new_clearing_tensor).  Only for rn <= nw (the plan refuses wider filters)."""
    kw, kx, nw, rn = nd.dims[:4]
    u0, u1, u2 = nd.dims[4:7]
    assert rn <= nw
    P, n = nw * nw, x.shape[0]
    w = nd.weights.reshape(kw, kx, rn, rn)
    xc = x.reshape(n, kx, P)
    y = np.zeros((n, kw, P), dtype=np.int64)
    for c in range(kx):
        for a in range(rn):
            for b in range(rn):
                d = a * nw + b
                if d >= P or not w[:, c, a, b].any():
                    continue
                sh = np.zeros((n, P), dtype=np.int64)
                sh[:, : P - d] = xc[:, c, d:]
                y += w[:, c, a, b][None, :, None] * sh[:, None, :]
    if nd.bias is not None:
        y += nd.bias[None, :, None]
    o, i, j = np.meshgrid(np.arange(kw), np.arange(nw), np.arange(nw), indexing="ij")
    keep = ((o < u0) & (i < u1) & (j < u2)).reshape(kw, P)
    return np.where(keep[None], y, 0).reshape(n, -1)


def ref_forward(nodes, xs):
    """(outputs [n, out_len] int64, error bits [n], per-input output shape) of the node stack on the inputs xs [n, input_len]"""
    x = np.array(xs, dtype=np.int64, ndmin=2)
    n = x.shape[0]
    bad = _any((x < -128) | (x > 127))
    err = np.where(bad, 16, 0).astype(np.int64)
    x[bad] = 0                                       # an input outside the 8-bit domain is computed as zeros
    shape = (x.shape[1],)
    for nd in nodes:
        if nd.kind == DENSE:
            N, K = nd.dims[:2]
            x = x @ nd.weights.reshape(N, K).T
            if nd.bias is not None:
                x = x + nd.bias[None]
            shape = (N,)
        elif nd.kind == MATMUL:
            R, K, Cc, tr = nd.dims[:4]
            B = nd.weights.reshape(Cc, K).T if tr else nd.weights.reshape(K, Cc)
            y = x.reshape(n, R, K) @ B
            if nd.bias is not None:
                y = y + nd.bias[None, None]
            x, shape = y.reshape(n, -1), (R, Cc)
        elif nd.kind == CONV:
            x, shape = ref_conv(x, nd), (nd.dims[0], nd.dims[2], nd.dims[2])
        elif nd.kind == REQUANT:
            x, e, _ = ref_requant(x, nd)
            err |= e
        elif nd.kind == RELU:
            err |= np.where(_any((x < -128) | (x > 127)), 4, 0)
            x = np.maximum(x, 0)
        elif nd.kind == POOL:
            c, h, w = nd.dims[:3]
            v = x.reshape(n, c, h // 2, 2, w // 2, 2)
            mx = v.max(axis=(3, 5))
            err |= np.where(_any(mx[:, :, :, None, :, None] - v > 255), 8, 0)
            x, shape = mx.reshape(n, -1), (c, h // 2, w // 2)
        else:
            raise ValueError("unknown kind %d" % nd.kind)
    return x, err.astype(np.uint32), shape


# ---- device harness -----------------------------------------------------------------------------------------------------
def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _plan(gpu, nodes, input_len):
    """dp_infer_plan: (return code, plan handle, message)"""
    arr = (InferNode * max(1, len(nodes)))()
    for i, nd in enumerate(nodes):
        s = arr[i]
        s.kind = nd.kind
        for k, d in enumerate(nd.dims):
            s.dims[k] = d
        s.shift, s.clamp_size, s.intermediate_bits, s.multiplier = nd.shift, nd.clamp_size, nd.intermediate_bits, nd.multiplier
        s.weights = None if nd.weights is None else nd.weights.ctypes.data
        s.bias = None if nd.bias is None else nd.bias.ctypes.data
    h = C.c_void_p()
    rc = gpu.lib().dp_infer_plan(C.cast(arr, C.c_void_p), len(nodes), input_len, C.byref(h))
    return rc, h, (gpu.lib().dp_last_error().decode() if rc else "")


def _infer(gpu, nodes, xs, out_len):
    """(outputs, error bits, kernel launches of the run) from one plan and one dp_infer_run over the whole batch"""
    xs = np.ascontiguousarray(xs, dtype=np.int64)
    rc, h, msg = _plan(gpu, nodes, xs.shape[1])
    assert rc == gpu.DP_OK, msg
    try:
        out = np.zeros((xs.shape[0], out_len), dtype=np.int64)
        err = np.zeros(xs.shape[0], dtype=np.uint32)
        before = gpu.lib().dp_kernel_launches()
        gpu.check(gpu.lib().dp_infer_run(h, _ptr(xs), xs.shape[0], _ptr(out), _ptr(err)))
        return out, err, gpu.lib().dp_kernel_launches() - before
    finally:
        gpu.lib().dp_infer_free(h)


def assert_same(name, got, want, got_err, want_err, shape):
    """word for word, naming the first (input, element) that differs"""
    if not np.array_equal(got, want):
        j, i = (int(v) for v in np.argwhere(got != want)[0])
        idx = np.unravel_index(i, shape)
        pytest.fail("%s: input %d, element %s of %s: got %d, want %d (%d of %d words differ)"
                    % (name, j, tuple(int(v) for v in idx), shape, got[j, i], want[j, i], int((got != want).sum()), got.size))
    if not np.array_equal(got_err, want_err):
        j = int(np.argwhere(got_err != want_err)[0, 0])
        pytest.fail("%s: input %d: error bits %#x, want %#x (inputs with bits: got %s, want %s)"
                    % (name, j, got_err[j], want_err[j], np.flatnonzero(got_err).tolist(), np.flatnonzero(want_err).tolist()))


def check_on_device(gpu, name, nodes, xs, launches=None):
    want, want_err, shape = ref_forward(nodes, xs)
    got, got_err, ran = _infer(gpu, nodes, xs, want.shape[1])
    assert_same(name, got, want, got_err, want_err, shape)
    if launches is not None:
        base = _infer(gpu, [], xs, xs.shape[1])[2]     # the run's own launches (its stream sync) without any stage
        assert ran - base == launches, "%s: %d kernel launches, want %d" % (name, ran - base, launches)


# ---- case data ----------------------------------------------------------------------------------------------------------
def _rng(name):
    return np.random.Generator(np.random.PCG64(zlib.crc32(name.encode())))


def _values(rng, mode, shape):
    """'rand': uniform int8; 'ext': every value -128 or 127; 'onehot' (inputs): one entry of 1, -128 or 127 per input"""
    if mode == "ext":
        return rng.choice(np.array([-128, 127]), size=shape).astype(np.int64)
    if mode == "onehot":
        n, m = shape
        x = np.zeros(shape, dtype=np.int64)
        x[np.arange(n), (np.arange(n) * 7 + 3) % m] = np.array([1, -128, 127])[np.arange(n) % 3]
        return x
    return rng.integers(-128, 128, size=shape).astype(np.int64)


def _epilogue(gemm_nodes, xs, epi):
    """'gemm': store int32; 'rq' / 'rq_relu': + a fused Requant (and Relu) scaled so that the int8 outputs reach both clamps"""
    if epi == "gemm":
        return gemm_nodes
    v = np.abs(ref_forward(gemm_nodes, xs)[0]).max()
    shift = 20
    rq = requant(shift, 40, 31, max(1, int(round(300 * (1 << shift) / max(1, v)))))
    return gemm_nodes + [rq] + ([relu()] if epi == "rq_relu" else [])


# (N, K, batch, values, epilogue)
DENSE_CASES = [
    (1, 1, 1, "ext", "gemm"), (7, 3, 63, "rand", "rq"), (8, 31, 64, "onehot", "rq_relu"), (63, 32, 65, "ext", "rq"),
    (64, 33, 129, "rand", "gemm"), (65, 100, 1, "onehot", "gemm"), (129, 1024, 65, "rand", "rq_relu"),
    (129, 33, 129, "ext", "rq_relu"), (65, 1024, 64, "ext", "gemm"), (64, 100, 63, "onehot", "rq"),
    (8, 1024, 129, "onehot", "gemm"), (63, 3, 1, "rand", "rq_relu"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,n,vals,epi", DENSE_CASES, ids=["dense-N%d-K%d-n%d-%s-%s" % c for c in DENSE_CASES])
def test_dense(gpu, N, K, n, vals, epi):
    name = "dense-N%d-K%d-n%d-%s-%s" % (N, K, n, vals, epi)
    rng = _rng(name)
    w = _values(rng, "ext" if vals == "ext" else "rand", (N, K))
    b = rng.integers(-(1 << 20), 1 << 20, size=N)
    xs = _values(rng, vals, (n, K))
    check_on_device(gpu, name, _epilogue([dense(w, b)], xs, epi), xs)


# (R, K, C, transposed, bias, batch, values, epilogue); MODE 1 when K % 4 != 0
MATMUL_CASES = [
    (1, 1, 1, 0, 0, 1, "ext", "gemm"), (3, 2, 5, 1, 1, 22, "rand", "rq"), (17, 3, 64, 0, 1, 4, "onehot", "gemm"),
    (1, 5, 70, 1, 0, 65, "rand", "rq_relu"), (3, 36, 1, 0, 0, 21, "ext", "gemm"), (17, 64, 70, 1, 1, 8, "rand", "rq"),
    (17, 5, 5, 0, 1, 7, "ext", "rq_relu"), (3, 3, 70, 1, 0, 43, "onehot", "gemm"), (1, 64, 64, 0, 1, 64, "onehot", "rq"),
    (1, 2, 1, 1, 1, 129, "rand", "gemm"), (3, 1, 64, 1, 1, 5, "ext", "rq"), (17, 36, 5, 1, 0, 3, "rand", "rq_relu"),
    # bufend: R K is a multiple of 32 and the input is the largest tensor, so the last input's last row ends where the chunk's
    # buffer does and the read past it (Kp - K bytes) lands in the buffer's slack
    (8, 36, 5, 0, 1, 64, "rand", "gemm"), (32, 5, 1, 1, 0, 65, "ext", "gemm"),
]


def _mm_id(c):
    R, K, Cc, tr, b, n, vals, epi = c
    return "mm-mode%d-R%d-K%d-C%d-%s-%s-n%d-%s-%s%s" % (0 if K % 4 == 0 else 1, R, K, Cc, "T" if tr else "N", "bias" if b else "nobias",
                                                       n, vals, epi, "-bufend" if R * K % 32 == 0 and K % 32 != 0 else "")


@pytest.mark.gpu
@pytest.mark.parametrize("case", MATMUL_CASES, ids=[_mm_id(c) for c in MATMUL_CASES])
def test_matmul(gpu, case):
    R, K, Cc, tr, has_bias, n, vals, epi = case
    name = _mm_id(case)
    rng = _rng(name)
    stored = _values(rng, "ext" if vals == "ext" else "rand", (Cc, K) if tr else (K, Cc))
    b = rng.integers(-(1 << 20), 1 << 20, size=Cc) if has_bias else None
    xs = _values(rng, vals, (n, R * K))
    check_on_device(gpu, name, _epilogue([matmul(R, K, Cc, stored, tr, b)], xs, epi), xs)


# (nw, kx, rn, kw, (u0, u1, u2), batch, values, epilogue, filter): 'prune' zeroes some taps in every output channel, 'zero' all
CONV_CASES = [
    (4, 1, 3, 3, (2, 2, 1), 9, "rand", "rq_relu", "prune"), (4, 4, 1, 70, (69, 4, 3), 5, "ext", "gemm", "prune"),
    (8, 3, 5, 1, (1, 4, 3), 3, "onehot", "gemm", "prune"), (16, 1, 5, 70, (65, 12, 9), 2, "rand", "rq", "prune"),
    (32, 3, 3, 3, (2, 30, 29), 3, "ext", "rq_relu", "prune"), (8, 4, 3, 70, (70, 6, 5), 4, "rand", "gemm", "dense"),
    (4, 3, 3, 3, (2, 3, 2), 17, "ext", "rq", "prune"), (16, 4, 5, 3, (3, 16, 15), 2, "onehot", "rq_relu", "prune"),
    (4, 3, 3, 3, (2, 3, 1), 9, "rand", "gemm", "zero"), (8, 1, 3, 70, (5, 7, 2), 6, "ext", "rq_relu", "zero"),
]


def _conv_id(c):
    nw, kx, rn, kw, u, n, vals, epi, filt = c
    return "conv-nw%d-P%d-kx%d-rn%d-kw%d-u%d.%d.%d-n%d-%s-%s-%s%s" % (nw, nw * nw, kx, rn, kw, u[0], u[1], u[2], n, vals, epi, filt,
                                                                    "-K0" if filt == "zero" else "")


def _conv_filter(rng, kw, kx, rn, vals, mode):
    f = _values(rng, "ext" if vals == "ext" else "rand", (kw, kx, rn, rn))
    if mode == "zero":
        return np.zeros_like(f)
    if mode == "prune":                      # about a third of the taps zero in every output channel, at least one kept
        dead = rng.random(kx * rn * rn) < 0.35
        dead[rng.integers(kx * rn * rn)] = False
        f.reshape(kw, -1)[:, dead] = 0
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONV_CASES, ids=[_conv_id(c) for c in CONV_CASES])
def test_conv(gpu, case):
    nw, kx, rn, kw, u, n, vals, epi, mode = case
    name = _conv_id(case)
    rng = _rng(name)
    f = _conv_filter(rng, kw, kx, rn, vals, mode)
    b = rng.integers(-(1 << 20), 1 << 20, size=kw)
    xs = _values(rng, vals, (n, kx * nw * nw))
    nodes = _epilogue([conv(f, b, nw, u)], xs, epi)
    if mode == "zero":                       # K = 0 after pruning: the bias on kept positions, 0 elsewhere
        want = ref_forward(nodes[:1], xs)[0].reshape(n, kw, nw, nw)
        assert (want[:, : u[0], : u[1], : u[2]] == b[: u[0], None, None]).all() and want.sum() == n * u[1] * u[2] * b[: u[0]].sum()
    check_on_device(gpu, name, nodes, xs)


# ---- the exactness bound ------------------------------------------------------------------------------------------------
EDGE_K = (1 << 17) - 1                      # Kp = 2^17: 4096 k-steps


def _edge_layer():
    """row 0: weights -128 against inputs of -128 reach 2^31 - 1 with bias 2^14 - 1; row 1: weights 127 reach -(2^31 - 1) with the
    bias that makes 128 sum|w| + |b| = 2^31 - 1 too"""
    w = np.stack([np.full(EDGE_K, -128), np.full(EDGE_K, 127)]).astype(np.int64)
    b = np.array([I32_MAX - 128 * 128 * EDGE_K, -(I32_MAX - 128 * 127 * EDGE_K)], dtype=np.int64)
    assert (128 * np.abs(w).sum(axis=1) + np.abs(b) == I32_MAX).all()
    return w, b


@pytest.mark.gpu
def test_exactness_bound_edge(gpu):
    w, b = _edge_layer()
    xs = np.stack([np.full(EDGE_K, -128), np.full(EDGE_K, 127), _rng("edge").integers(-128, 128, size=EDGE_K)]).astype(np.int64)
    want = ref_forward([dense(w, b)], xs)[0]
    assert want[0].tolist() == [I32_MAX, -I32_MAX]
    check_on_device(gpu, "dense-edge-K131071-bound", [dense(w, b)], xs, launches=1)
    for row, delta in ((0, 1), (1, -1)):      # one past the bound on either row is refused, naming the node and the row
        b2 = b.copy()
        b2[row] += delta
        rc, h, msg = _plan(gpu, [relu(), dense(w, b2)], EDGE_K)
        assert rc == gpu.DP_ERR_INVALID and not h.value, msg
        assert "node 1 " in msg and ("output %d " % row) in msg and "exceed int32" in msg, msg


# ---- element-wise stages, Requant edges and fusion -----------------------------------------------------------------------
def _small_dense(rng, N, K):
    """weights in [-6, 6]: outputs of full-range inputs reach a few thousand"""
    return dense(rng.integers(-6, 7, size=(N, K)), rng.integers(-20, 21, size=N))


def _gather_dense(rng, N, K, bias=None):
    """one weight of 1 per row: output r is input[k_r] (+ bias[r]), so an int32 Relu / Maxpool after it sees the 8-bit range"""
    w = np.zeros((N, K), dtype=np.int64)
    w[np.arange(N), rng.integers(0, K, size=N)] = 1
    return dense(w, bias)


def _tie_rq():
    """m = 1, shift = 1: cl = (v + 1) >> 1 -- a tie on every odd v, both clamps beyond |v| = 255"""
    return requant(1, 16, 20, 1)


def _stack(name):
    """(nodes, inputs, the launches the plan should take)"""
    rng = _rng(name)
    xs = _values(rng, "rand", (70, 64))
    xs[::5, ::3] = -128
    xs[1::5, 1::3] = 127
    if name == "empty":                                  # no nodes: the output is the input
        return [], xs, 0
    if name == "dense-rq-relu-dense":
        d1 = dense(rng.integers(-128, 128, size=(32, 64)), rng.integers(-999, 1000, size=32))
        d2 = dense(rng.integers(-128, 128, size=(10, 32)), None)
        return _epilogue([d1], xs, "rq_relu") + [d2], xs, 2
    if name == "dense-relu":                             # the GEMM stores int32, Relu runs on it
        return [_gather_dense(rng, 16, 64), relu()], xs, 2
    if name == "dense-relu-pool-rq-int32":               # every element-wise kernel on int32
        return [_gather_dense(rng, 64, 64), relu(), pool(4, 4, 4), requant(2, 16, 20, 3)], xs, 4
    if name == "dense-pool-rq-ties-int32":               # +-300 on each pooled channel: both clamps, windows within 255
        return [_gather_dense(rng, 32, 64, np.repeat([300, -300], 16)), pool(2, 4, 4), _tie_rq()], xs, 3
    if name == "dense-rq-ties-fused":
        return [_small_dense(rng, 33, 64), _tie_rq()], xs, 1
    if name == "dense-rq-pool-relu-int8":                # fused Requant, then Maxpool and Relu on int8
        return [_small_dense(rng, 64, 64), _tie_rq(), pool(4, 4, 4), relu()], xs, 3
    if name == "rq-relu-pool-dense-int8":                # element-wise kernels on the int8 model input, then the GEMM
        return [requant(1, 9, 7, 3), relu(), pool(1, 8, 8), dense(rng.integers(-128, 128, size=(5, 16)), None)], xs, 4
    if name == "conv-rq-relu-pool":
        f = _conv_filter(rng, 4, 1, 3, "rand", "prune")
        return _epilogue([conv(f, rng.integers(-99, 100, size=4), 8, (3, 6, 5))], xs, "rq_relu") + [pool(4, 8, 8)], xs, 2
    if name == "mm-rq-relu-mm-rq":
        m1 = matmul(8, 8, 6, rng.integers(-128, 128, size=(8, 6)), 0, rng.integers(-99, 100, size=6))
        nodes = _epilogue([m1], xs, "rq_relu")
        m2 = matmul(8, 6, 3, rng.integers(-128, 128, size=(3, 6)), 1, None)
        return nodes + [m2, requant(14, 20, 31, 1 << 6)], xs, 2
    raise KeyError(name)


STACKS = ["empty", "dense-rq-relu-dense", "dense-relu", "dense-relu-pool-rq-int32", "dense-pool-rq-ties-int32", "dense-rq-ties-fused",
          "dense-rq-pool-relu-int8", "rq-relu-pool-dense-int8", "conv-rq-relu-pool", "mm-rq-relu-mm-rq"]


def test_stacks_reach_requant_edges():
    """CPU: the tie stacks' Requant inputs reach both clamps and rounding ties, and the stacks' inputs are in the domain"""
    for name in ("dense-pool-rq-ties-int32", "dense-rq-ties-fused"):
        nodes, xs, _ = _stack(name)
        v = ref_forward(nodes[:-1], xs)[0]
        _, err, cl = ref_requant(v, nodes[-1])
        assert (cl > 127).any() and (cl < -127).any() and (v % 2 == 1).any(), name
        assert (v < 0).any() and (err == 0).all(), name
    for name in STACKS:
        nodes, xs, _ = _stack(name)
        assert (ref_forward(nodes, xs)[1] == 0).all(), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", STACKS)
def test_stack_and_fusion(gpu, name):
    """outputs and bits equal the reference, and the run takes exactly the stages the plan should build (a Requant right after a
    GEMM, and a Relu right after that, run in its epilogue; everything else is its own launch)"""
    nodes, xs, launches = _stack(name)
    check_on_device(gpu, name, nodes, xs, launches)


# ---- per-input error bits in shared tiles ---------------------------------------------------------------------------------
N_ERR = 24                                  # MatMul R = 3: 72 GEMM rows, input 21 straddles the first M tile; Conv P = 16: 6 tiles
FAILING = [1, 4, 7, 10, 13, 16, 19, 21, 23]


def _err_inputs(rng, length, rows, alternate):
    """passing inputs in [-1, 1] (with -128 / 127 where bit 16 is tested); failing ones large, one sign per input (per row when
    `alternate`, so that a Maxpool window mixes signs)"""
    xs = rng.integers(-1, 2, size=(N_ERR, length)).astype(np.int64)
    for j in FAILING:
        sign = np.where(np.arange(rows) % 2 == 1, -1, 1) if alternate else np.full(rows, 1 if j % 2 else -1)
        xs[j] = (rng.integers(64, 128, size=(rows, length // rows)) * sign[:, None]).reshape(-1)
    return xs


def _err_case(name):
    """(nodes, inputs, the bit only the FAILING inputs raise)"""
    rng = _rng(name)
    layer, bit = name.split("-")[:2], int(name.split("bit")[1])
    if layer[0] == "mm":                    # R = 3, K = 5 (MODE 1), C = 4; weights in [1, 8]: |v| <= 44 passing, >= 316 failing
        gemm = matmul(3, 5, 4, rng.integers(1, 9, size=(5, 4)), 0, rng.integers(-4, 5, size=4))
        length, rows, pool_shape = 15, 3, (1, 2, 6)   # the pool's windows take two columns of two rows
    else:                                   # nw = 4 (P = 16), kx = 1, rn = 3, kw = 2; column 1 cleared, so each window holds a 0
        gemm = conv(rng.integers(1, 9, size=(2, 1, 3, 3)), rng.integers(-4, 5, size=2), 4, (2, 3, 1))
        length, rows, pool_shape = 16, 1, (2, 4, 4)
    xs = _err_inputs(rng, length, rows, alternate=bit == 8)
    if bit == 1:
        nodes = [gemm, requant(1, 15, 7, 1)]            # |v| > 2^7
    elif bit == 2:
        nodes = [gemm, requant(1, 8, 20, 1)]            # cl = (v + 1) >> 1 outside [-128, 128)
    elif bit == 4:
        nodes = [gemm, relu()]                          # Relu on int32 outside [-128, 127]
    elif bit == 8:
        nodes = [gemm, pool(*pool_shape)]               # Maxpool on int32: max - v > 255
    else:                                               # 128 / -129 in the failing inputs, -128 and 127 in the passing ones
        xs = rng.integers(-128, 128, size=(N_ERR, length)).astype(np.int64)
        xs[:, 0], xs[:, -1] = -128, 127
        for k, j in enumerate(FAILING):
            xs[j, (3 * k) % length] = 128 if k % 2 else -129
        nodes = [gemm, requant(10, 16, 20, 5)]
    return nodes, xs, bit


ERROR_CASES = ["%s-bit%d" % (layer, bit) for layer in ("mm-R3", "conv-P16") for bit in (1, 2, 4, 8, 16)]


@pytest.mark.parametrize("name", ERROR_CASES)
def test_error_cases_fail_where_intended(name):
    """CPU: in the reference, exactly the FAILING inputs raise exactly the case's bit"""
    nodes, xs, bit = _err_case(name)
    err = ref_forward(nodes, xs)[1]
    want = np.zeros(N_ERR, dtype=np.uint32)
    want[FAILING] = bit
    assert err.tolist() == want.tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ERROR_CASES)
def test_error_bits_per_input(gpu, name):
    """the failing inputs carry the bit and only they do; every input's outputs (the failing ones' too) equal the reference"""
    nodes, xs, _ = _err_case(name)
    check_on_device(gpu, name, nodes, xs)


# ---- plan refusals ---------------------------------------------------------------------------------------------------------
def _refusal(name):
    """(nodes, input_len, the node the message must name, a fragment of the message)"""
    rng = _rng(name)
    d16 = dense(rng.integers(-128, 128, size=(16, 64)), None)
    f = rng.integers(-128, 128, size=(2, 1, 3, 3))
    if name == "unknown-kind":
        return [d16, Node(6)], 64, 1, "unknown kind"
    if name == "maxpool-shape":
        return [d16, pool(1, 4, 2)], 64, 1, "shape does not match"
    if name == "maxpool-odd":
        return [d16, pool(4, 1, 4)], 64, 1, "shape does not match"
    if name == "conv-nw-not-pow2":
        return [conv(f, None, 6, (2, 4, 4))], 36, 0, "shape does not match"
    if name == "conv-shape":
        return [conv(f, None, 8, (2, 6, 6))], 128, 0, "shape does not match"
    if name == "conv-filter-wider-than-image":        # rn = 5 > nw = 4: the FFT convolution would drop the taps b >= nw
        return [conv(rng.integers(-128, 128, size=(2, 1, 5, 5)), None, 4, (2, 4, 4))], 16, 0, "exceeds the padded image width 4"
    if name == "matmul-shape":
        return [matmul(3, 5, 4, rng.integers(-128, 128, size=20), 0)], 16, 0, "shape does not match"
    if name == "dense-ncols":
        return [dense(rng.integers(-128, 128, size=(4, 63)))], 64, 0, "ncols does not match"
    if name == "requant-shift0":
        return [d16, requant(0, 16, 20, 1)], 64, 1, "shift and clamping size"
    if name == "requant-shift63":
        return [requant(63, 16, 20, 1)], 64, 0, "shift and clamping size"
    if name == "requant-intermediate63":
        return [d16, relu(), requant(8, 16, 63, 1)], 64, 2, "intermediate bits"
    if name == "weight-minus129":
        w = rng.integers(-128, 128, size=(16, 64))
        w[5, 7] = -129
        return [relu(), dense(w)], 64, 1, "weight -129 outside [-128, 127]"
    if name == "bias-outside-int32":
        return [dense(np.zeros((4, 64), dtype=np.int64), [0, 0, 1 << 31, 0])], 64, 0, "bias 2147483648 outside int32"
    if name == "not-8-bit":
        return [d16, relu(), dense(rng.integers(-128, 128, size=(4, 16)))], 64, 2, "not 8-bit"
    raise KeyError(name)


REFUSALS = ["unknown-kind", "maxpool-shape", "maxpool-odd", "conv-nw-not-pow2", "conv-shape", "conv-filter-wider-than-image",
            "matmul-shape", "dense-ncols", "requant-shift0", "requant-shift63", "requant-intermediate63", "weight-minus129",
            "bias-outside-int32", "not-8-bit"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", REFUSALS)
def test_plan_refusals(gpu, name):
    nodes, input_len, node, fragment = _refusal(name)
    rc, h, msg = _plan(gpu, nodes, input_len)
    assert rc == gpu.DP_ERR_INVALID and not h.value, (rc, msg)
    assert ("node %d " % node) in msg or ("node %d:" % node) in msg, msg
    assert fragment in msg, msg


# ---- CPU: the reference pinned to the checker, and the node layout ---------------------------------------------------------
def _anchor(name):
    """(layer descriptors, weights, input) of a power-of-two stack the checker takes"""
    rng = _rng(name)
    if name == "dense-rq-relu":
        row, w, b = models.dense_layer(rng.integers(-127, 128, size=(24, 60)), rng.integers(-127, 128, size=24), np.arange(64) < 60, 32)
        desc = [row, models._requant(6, 2 * 7 + 6 + 1), [RELU] + [0] * 8]
        return desc, np.concatenate([w.reshape(-1), b]), rng.integers(-127, 128, size=64)
    if name.startswith("mm-"):
        tr, has_bias = "-T" in name, name.endswith("-bias")
        R, K, Cc = 4, 16, 8
        w = rng.integers(-127, 128, size=K * Cc)
        data = np.concatenate([w] + ([rng.integers(-999, 1000, size=Cc)] if has_bias else []))
        return [[MATMUL, R, K, Cc, int(tr), int(has_bias), 0, 0, 0]], data, rng.integers(-127, 128, size=R * K)
    # conv 3x3 (3 channels) over a 12x12 image in [4][16][16] -> requant -> relu -> maxpool
    row, filt, bias, h_out = models.conv_layer(rng.integers(-127, 128, size=(3, 3, 3, 3)), rng.integers(-1000, 1001, size=3), 16, 12)
    desc = [row, models._requant(7, 2 * 7 + 5), [RELU] + [0] * 8, [POOL, row[1], 16, 16, 0, 0, 0, 0, 0]]   # as models.cnn sizes it
    x = np.zeros((4, 16, 16), dtype=np.int64)
    x[:3, :12, :12] = rng.integers(-127, 128, size=(3, 12, 12))
    return desc, np.concatenate([filt.reshape(-1), bias]), x.reshape(-1)


ANCHORS = ["dense-rq-relu", "mm-N-nobias", "mm-N-bias", "mm-T-nobias", "mm-T-bias", "conv-rq-relu-pool"]


@pytest.mark.parametrize("name", ANCHORS)
def test_reference_equals_checker(name):
    desc, data, x = _anchor(name)
    nodes = nodes_from_desc(desc, data)
    out, err, _ = ref_forward(nodes, x[None])
    assert err.tolist() == [0]
    assert np.array_equal(out[0], M.model_output(desc, data, x))
    if name.startswith("conv"):             # the kept positions are the 2-D valid correlation of the real image, + bias
        nd = nodes[0]
        kw_u, h = nd.dims[4], nd.dims[5]
        y = ref_forward(nodes[:1], x[None])[0].reshape(nd.dims[0], 16, 16)
        img = x.reshape(4, 16, 16)[:3, :12, :12]
        filt = nd.weights.reshape(nd.dims[0], 4, 4, 4)[:, :3, :3, :3]
        for o in range(kw_u):
            want = signal.correlate(img, filt[o], mode="valid", method="direct")[0] + nd.bias[o]
            assert np.array_equal(y[o, :h, :h], want), "channel %d" % o
        assert not y[kw_u:].any() and not y[:, h:].any() and not y[:, :, h:].any()


def test_node_layout():
    """the ctypes copy of dp_infer_node matches the header's x86-64 layout: 72 bytes, the multiplier at 48; every field's offset as
    the C compiler lays it out"""
    assert C.sizeof(InferNode) == 72 and InferNode.multiplier.offset == 48
    cxx = os.environ.get("CXX") or shutil.which("g++") or shutil.which("c++")
    assert cxx, "no C++ compiler to read the header's layout"
    fields = [f for f, _ in InferNode._fields_]
    src = ('#include <cstdio>\n#include <cstddef>\n#include "deepprove_b200.h"\nint main() { printf("%zu", sizeof(dp_infer_node));'
           + "".join(' printf(" %%zu", offsetof(dp_infer_node, %s));' % f for f in fields) + " }\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "layout.cpp"), "w").write(src)
        subprocess.run([cxx, "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-o", os.path.join(d, "layout"), os.path.join(d, "layout.cpp")],
                       check=True)
        got = [int(v) for v in subprocess.run([os.path.join(d, "layout")], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(InferNode)] + [getattr(InferNode, f).offset for f in fields]
