"""Synthetic quantised models in the padded (power-of-two) layout the prover works in, as plain arrays: the layer
descriptor consumed by dph_model_context_new (host/capi.cpp) -- 9 int64 per node {kind, 8 shape words} plus the weights
in node order.  Pure numpy; both bench arms are fed the same arrays.

CNN-264k (SURVEY.md 8(d) Cfg 3): zkml/assets/scripts/CNN/cifar-cnn.py:175-241 with --num-params 264000 gives
c1 = 12, c2 = 33, fc1 = 247, fc2 = 173:  [3,32,32] -> conv5x5(12) -> requant -> relu -> maxpool -> conv5x5(33) -> requant
-> relu -> maxpool -> flatten(33*5*5) -> fc 247 -> requant -> relu -> fc 173 -> requant -> relu -> fc 10."""
import numpy as np

DENSE, REQUANT, RELU, CONV, POOL, MATMUL = 0, 1, 2, 3, 4, 5
BIT_LEN = 8


def _p2(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def _clog2(x):
    return int(x - 1).bit_length() if x > 1 else 0


def _requant(int_part_log, intermediate_bits):
    """layers/requant.rs:395-410 shape: shift = fp_scale + right_shift is a multiple of BIT_LEN, multiplier = 0.75 * 2^fp_scale"""
    fp = ((int_part_log + 24 + 7) // 8) * 8 - int_part_log
    return [REQUANT, int_part_log, fp, 3 << (fp - 2), intermediate_bits, 0, 0, 0, 0]


def conv_layer(filt_u, bias_u, n_p, n_u):
    """A Convolution node in the padded layout: filter [kw_u, kx_u, k, k] and bias [kw_u] over a [kx_u, n_u, n_u] image held in
    [p2(kx_u), n_p, n_p].  The filter is padded to [p2(kw_u), p2(kx_u), p2(k), p2(k)], the bias to p2(kw_u) (zeros).
    Returns (descriptor row, padded filter, padded bias, h_out = n_u - k + 1)."""
    kw_u, kx_u, k, _ = filt_u.shape
    kw, kx, rn = _p2(kw_u), _p2(kx_u), _p2(k)
    filt = np.zeros((kw, kx, rn, rn), dtype=np.int64)
    filt[:kw_u, :kx_u, :k, :k] = filt_u
    bias = np.zeros(kw, dtype=np.int64)
    bias[:kw_u] = bias_u
    h_out = n_u - k + 1
    return [CONV, kw, kx, n_p, rn, kw_u, h_out, h_out, 0], filt, bias, h_out


def flatten_mask(c_u, n_u, n_p):
    """The real columns of a flatten of [p2(c_u)][n_p][n_p] (padding.rs pad_matrix_to_ignore_garbage): c < c_u, row < n_u, col < n_u"""
    mask = np.zeros((_p2(c_u), n_p, n_p), dtype=bool)
    mask[:c_u, :n_u, :n_u] = True
    return mask.reshape(-1)


def dense_layer(w_u, b_u, real, nrows):
    """A Dense node in the padded layout: the [out_u, real.sum()] matrix spread over the columns where `real` is True (zeros
    elsewhere) and over the first out_u of `nrows` rows, the bias likewise.  Returns (descriptor row, padded matrix, padded bias)."""
    out_u = w_u.shape[0]
    w = np.zeros((nrows, real.size), dtype=np.int64)
    w[:out_u, real] = w_u
    b = np.zeros(nrows, dtype=np.int64)
    b[:out_u] = b_u
    return [DENSE, nrows, real.size, 0, 0, 0, 0, 0, 0], w, b


def cnn(seed=1, img=32, c0=3, c1=12, c2=33, f1=247, f2=173, f3=10, k=5):
    """returns (desc [n_nodes, 9] int64, data int64, input int64 [padded c0 * img^2], n_real_params)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    desc, data, n_params = [], [], 0
    kx_u, n_u, n_p = c0, img, _p2(img)
    x = np.zeros((_p2(c0), n_p, n_p), dtype=np.int64)
    x[:c0, :img, :img] = rng.integers(-127, 128, size=(c0, img, img))
    for kw_u in (c1, c2):
        filt_u = rng.integers(-127, 128, size=(kw_u, kx_u, k, k))
        row, filt, bias, h_out = conv_layer(filt_u, rng.integers(-1000, 1001, size=kw_u), n_p, n_u)
        kw = row[1]
        n_params += kw_u * kx_u * k * k + kw_u
        desc.append(row)
        data += [filt.reshape(-1), bias]
        terms = k * k * kx_u
        desc.append(_requant(_clog2(terms) + 2, 2 * (BIT_LEN - 1) + _clog2(terms + 1)))   # convolution.rs:362-366 output_bitsize
        desc.append([RELU] + [0] * 8)
        desc.append([POOL, kw, n_p, n_p, 0, 0, 0, 0, 0])
        kx_u, n_u, n_p = kw_u, h_out // 2, n_p // 2
    ncols, prev_real = _p2(c2) * n_p * n_p, None
    for li, out_u in enumerate((f1, f2, f3)):
        nrows = _p2(out_u)
        real = flatten_mask(c2, n_u, n_p) if li == 0 else np.arange(ncols) < prev_real
        w_u = rng.integers(-127, 128, size=(out_u, int(real.sum())))
        row, w, b = dense_layer(w_u, rng.integers(-127, 128, size=out_u), real, nrows)
        n_params += out_u * int(real.sum()) + out_u
        desc.append(row)
        data += [w.reshape(-1), b]
        if li < 2:
            desc.append(_requant(_clog2(ncols), 2 * (BIT_LEN - 1) + _clog2(ncols) + 1))   # dense.rs:416-421
            desc.append([RELU] + [0] * 8)
        ncols, prev_real = nrows, out_u
    return np.asarray(desc, dtype=np.int64), np.concatenate(data).astype(np.int64), x.reshape(-1), n_params


def cnn_small(seed=1):
    return cnn(seed, img=16, c0=3, c1=4, c2=6, f1=24, f2=16, f3=10, k=3)


def covid(seed=1, img=224, channels=(32, 64, 64, 128, 128), fc=64, k=3):
    """The reference's vision model (zkml/assets/scripts/covid/covid.py, CNNModel.forward) in the padded layout, same rules as
    cnn():  [3,img,img] -> conv(c1) -> requant -> relu -> conv(c2) -> requant -> relu -> maxpool -> [conv -> requant -> relu
    -> maxpool] x 3 -> flatten -> dense fc -> requant -> relu -> dense 1 -> requant -> relu.  Dropout is the identity at
    inference.  The one-output dense layer is padded to 4 rows (rows 2-4 and their bias are zero): the requant and ReLU
    lookups that follow it need tensors of at least 4 entries (their LogUp circuits refuse a 2-entry column).  At img = 224
    the padded widths are 256, 256, 128, 64, 32 (FFT rows of 2^17, 2^17, 2^15, 2^13, 2^11).
    Returns (desc, data, input, n_real_params); the defaults have 1,457,537 real parameters."""
    rng = np.random.Generator(np.random.PCG64(seed))
    desc, data, n_params = [], [], 0
    c0 = 3
    kx_u, n_u, n_p = c0, img, _p2(img)
    x = np.zeros((_p2(c0), n_p, n_p), dtype=np.int64)
    x[:c0, :img, :img] = rng.integers(-127, 128, size=(c0, img, img))
    for li, kw_u in enumerate(channels):
        filt_u = rng.integers(-127, 128, size=(kw_u, kx_u, k, k))
        row, filt, bias, h_out = conv_layer(filt_u, rng.integers(-1000, 1001, size=kw_u), n_p, n_u)
        kw = row[1]
        n_params += kw_u * kx_u * k * k + kw_u
        desc.append(row)
        data += [filt.reshape(-1), bias]
        terms = k * k * kx_u
        desc.append(_requant(_clog2(terms) + 2, 2 * (BIT_LEN - 1) + _clog2(terms + 1)))
        desc.append([RELU] + [0] * 8)
        kx_u, n_u = kw_u, h_out
        if li > 0:                                  # conv1 feeds conv2 directly
            desc.append([POOL, kw, n_p, n_p, 0, 0, 0, 0, 0])
            n_u, n_p = n_u // 2, n_p // 2
    ncols, prev_real = _p2(kx_u) * n_p * n_p, None
    for li, out_u in enumerate((fc, 1)):
        nrows = max(4, _p2(out_u))
        real = flatten_mask(kx_u, n_u, n_p) if li == 0 else np.arange(ncols) < prev_real
        w_u = rng.integers(-127, 128, size=(out_u, int(real.sum())))
        row, w, b = dense_layer(w_u, rng.integers(-127, 128, size=out_u), real, nrows)
        n_params += out_u * int(real.sum()) + out_u
        desc.append(row)
        data += [w.reshape(-1), b]
        desc.append(_requant(_clog2(ncols), 2 * (BIT_LEN - 1) + _clog2(ncols) + 1))
        desc.append([RELU] + [0] * 8)
        ncols, prev_real = nrows, out_u
    return np.asarray(desc, dtype=np.int64), np.concatenate(data).astype(np.int64), x.reshape(-1), n_params


_KIND_NAMES = {DENSE: "Dense", REQUANT: "Requant", RELU: "ReLU", CONV: "Conv", POOL: "Maxpool2D", MATMUL: "MatMul"}


def stack_rows(desc, data, input_len, rows):
    """The model that proves `rows` inputs of (desc, data, input_len) at once, as the rows of one input matrix (the reference's MatMul
    with OperandMatrix::Input x OperandMatrix::Weight, zkml/src/layers/matrix_mul.rs).  With R = p2(rows): a Dense {nrows, ncols}
    becomes MatMul {R, ncols, nrows, TransposeB, bias} -- its [nrows][ncols] weights are the [C][K] right matrix and its bias the
    MatMul bias, so `data` is returned unchanged -- and a MatMul {r, k, c, t, b} becomes {R*r, k, c, t, b}; Requant and ReLU work
    element by element and stay.  Row r of the stacked input ([R][input_len], row-major) is input r in the base model's padded
    layout, and row r of the stacked output ([R][output_len]) is that input's output.  Returns (desc', data, R * input_len, R).
    Raises ValueError for rows < 1, a Conv or Maxpool2D node (the reference's Convolution takes one image), an unknown node kind,
    or nodes whose shapes do not chain."""
    d = np.asarray(desc, dtype=np.int64).reshape(-1, 9)
    if int(rows) < 1:
        raise ValueError("stack_rows: rows must be at least 1, got %d" % int(rows))
    R = _p2(int(rows))
    out = d.copy()
    cur = int(input_len)                       # elements of one input row's tensor before node i
    for i, row in enumerate(d):
        kind = int(row[0])
        name = _KIND_NAMES.get(kind, "kind %d" % kind)
        if kind in (CONV, POOL):
            raise ValueError("stack_rows: node %d (%s) does not stack: the reference's Convolution and Maxpool2D take one image" % (i, name))
        if kind == DENSE:
            nrows, ncols = int(row[1]), int(row[2])
            if ncols != cur:
                raise ValueError("stack_rows: node %d (%s) takes %d inputs but follows a tensor of %d" % (i, name, ncols, cur))
            out[i] = [MATMUL, R, ncols, nrows, 1, 1, 0, 0, 0]
            cur = nrows
        elif kind == MATMUL:
            r, k, c = int(row[1]), int(row[2]), int(row[3])
            if r * k != cur:
                raise ValueError("stack_rows: node %d (%s) takes a [%d][%d] matrix but follows a tensor of %d" % (i, name, r, k, cur))
            out[i, 1] = R * r
            cur = r * c
        elif kind not in (REQUANT, RELU):
            raise ValueError("stack_rows: node %d has an unknown kind (%s)" % (i, name))
    return out, data, R * int(input_len), R


def pad_rows(xs, R):
    """The input of one stacked proof: m <= R inputs ([m, input_len]) as the first m rows of an [R][input_len] matrix, the rest filled
    with copies of the last input, flattened row-major.  Copies, not zeros: an input that passed screening cannot fail a lookup,
    while nothing keeps a zero row's outputs (the bias chain) inside the tables."""
    xs = np.asarray(xs, dtype=np.int64)
    if xs.ndim != 2 or not 1 <= xs.shape[0] <= R:
        raise ValueError("pad_rows: expected [1..%d, input_len] inputs, got shape %s" % (R, xs.shape))
    return np.concatenate([xs, np.repeat(xs[-1:], R - xs.shape[0], axis=0)]).reshape(-1)


def token_mlp(seed=1, tokens=8, d_model=64, d_hidden=128, transposed=(False, True), bias=(True, False)):
    """A token-wise MLP as the transformer feed-forward block uses it (zkml/src/layers/matrix_mul.rs: OperandMatrix::Input x
    OperandMatrix::Weight): X [tokens, d_model] -> MatMul(W1 [d_model, d_hidden] or its transpose, + bias) -> requant -> relu
    -> MatMul(W2 [d_hidden, d_model]) .  All dimensions powers of two (the padded layout).  Returns (desc, data, input)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    desc, data = [], []
    x = rng.integers(-127, 128, size=(tokens, d_model)).astype(np.int64)
    dims = [(d_model, d_hidden), (d_hidden, d_model)]
    for li, (k, c) in enumerate(dims):
        w = rng.integers(-127, 128, size=(k, c)).astype(np.int64)
        stored = w.T.copy() if transposed[li] else w          # Config::TransposeB keeps the matrix as [C][K]
        desc.append([MATMUL, tokens, k, c, int(transposed[li]), int(bias[li]), 0, 0, 0])
        data.append(stored.reshape(-1))
        if bias[li]:
            data.append(rng.integers(-127, 128, size=c).astype(np.int64))
        if li == 0:
            desc.append(_requant(_clog2(k), 2 * (BIT_LEN - 1) + _clog2(k) + 1))
            desc.append([RELU] + [0] * 8)
    return np.asarray(desc, dtype=np.int64), np.concatenate(data).astype(np.int64), x.reshape(-1)
