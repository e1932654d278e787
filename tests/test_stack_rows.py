"""Stacked models (models.stack_rows / pad_rows) on the CPU checker: many inputs of an MLP as the rows of the reference's Input x Weight
MatMul.  The descriptor transform keeps the weight data as it is, every refusal names its node, each row of the stacked model's output is
the base model's output of that row's input (copy-padded rows included), and the checker's stacked proofs are accepted by the restated
verifier against the true [R][N] output and rejected when one element of one row is changed."""
import os

import numpy as np
import pytest

import models
import onnx_import as I
import oracle_model_io as M
import oracle_py as O
from test_onnx_calibration import GOLDEN, samples

MATMUL, DENSE, REQUANT, RELU, CONV, POOL = models.MATMUL, models.DENSE, models.REQUANT, models.RELU, models.CONV, models.POOL


def mlp_2x64():
    """the 2x64 synthetic MLP as a layer descriptor, its data, and a source of distinct inputs"""
    w, b, rq = O.synthetic_mlp(2, 64, 5)
    desc = np.zeros((6, 9), dtype=np.int64)
    desc[0::3, 1:3] = 64
    desc[1::3, 0], desc[1::3, 1:5] = REQUANT, rq
    desc[2::3, 0] = RELU
    data = np.concatenate([w.reshape(2, -1), b.reshape(2, -1)], axis=1).reshape(-1)
    return desc, data, np.stack([O.synthetic_input(64, 6 + j) for j in range(8)])


def token_mlp():
    desc, data, x = models.token_mlp(seed=11, tokens=8, d_model=32, d_hidden=64)
    rng = np.random.Generator(np.random.PCG64(7))
    return desc, data, rng.integers(-127, 128, size=(8, x.size)).astype(np.int64)


def iris(calibrated):
    xs = samples("mlp-iris-01")[0]
    desc, data, _, md, _, _ = I.import_onnx(os.path.join(GOLDEN, "mlp-iris-01.onnx"), xs if calibrated else None)
    return desc, data, md.quantize_input(xs)


def dense_4m_desc():
    """Dense-4M's descriptor: 4 x [Dense 1024x1024 -> Requant -> ReLU] (bench.py DenseWorkload)"""
    desc = np.zeros((12, 9), dtype=np.int64)
    desc[0::3, 1:3] = 1024
    desc[1::3, 0], desc[1::3, 1:5] = REQUANT, [10, 22, 3 << 20, 25]
    desc[2::3, 0] = RELU
    return desc


MODELS = {"mlp_2x64": mlp_2x64, "token_mlp": token_mlp, "iris_absmax": lambda: iris(False), "iris_calibrated": lambda: iris(True)}


def _expected_desc(desc, R):
    want = desc.copy()
    for i, row in enumerate(desc):
        if row[0] == DENSE:
            want[i] = [MATMUL, R, row[2], row[1], 1, 1, 0, 0, 0]
        elif row[0] == MATMUL:
            want[i, 1] = R * row[1]
    return want


@pytest.mark.parametrize("rows", [1, 2, 5, 8, 30])
@pytest.mark.parametrize("name", list(MODELS) + ["dense_4m"])
def test_descriptor_transform(name, rows):
    if name == "dense_4m":
        desc, data, input_len = dense_4m_desc(), np.zeros(4 * (1024 * 1024 + 1024), dtype=np.int64), 1024
    else:
        desc, data, xs = MODELS[name]()
        input_len = xs.shape[1]
    before = desc.copy()
    sdesc, sdata, slen, R = models.stack_rows(desc, data, input_len, rows)
    assert R == models._p2(rows) and slen == R * input_len
    assert sdata is data, "the stacked model must reuse the base model's data as it is"
    assert np.array_equal(sdesc, _expected_desc(desc, R))
    assert np.array_equal(desc, before), "the base descriptor must not change"


def test_transposed_matmul_layout_is_dense_layout():
    """a Dense node's data (weights [nrows][ncols], then bias [nrows]) read as the stacked MatMul's (right matrix [C][K] under
    TransposeB, then bias [C]) computes the Dense layer on every row"""
    rng = np.random.default_rng(3)
    nrows, ncols, R = 8, 16, 4
    w, b = rng.integers(-127, 128, (nrows, ncols)), rng.integers(-127, 128, nrows)
    data = np.concatenate([w.reshape(-1), b])
    desc = np.array([[DENSE, nrows, ncols, 0, 0, 0, 0, 0, 0]], dtype=np.int64)
    sdesc, sdata, _, _ = models.stack_rows(desc, data, ncols, R)
    _, r, k, c, t, has_bias = sdesc[0, :6]
    right = sdata[: k * c].reshape(c, k) if t else sdata[: k * c].reshape(k, c).T
    bias = sdata[k * c: k * c + c] if has_bias else np.zeros(c, dtype=np.int64)
    xs = rng.integers(-127, 128, (r, k))
    assert np.array_equal(xs @ right.T + bias, np.stack([w @ x + b for x in xs]))


def test_cifar_refused_at_first_conv():
    for cal in (None, samples("cnn-cifar-01")[0]):
        desc, data, input_len = I.import_onnx(os.path.join(GOLDEN, "cnn-cifar-01.onnx"), cal)[:3]
        with pytest.raises(ValueError, match=r"node 0 \(Conv\)"):
            models.stack_rows(desc, data, input_len, 4)


def test_refusals():
    desc, data, xs = mlp_2x64()
    for rows in (0, -3):
        with pytest.raises(ValueError, match="rows must be at least 1"):
            models.stack_rows(desc, data, 64, rows)
    pool = np.concatenate([desc[:3], [[POOL, 4, 4, 4, 0, 0, 0, 0, 0]], desc[3:]])
    with pytest.raises(ValueError, match=r"node 3 \(Maxpool2D\)"):
        models.stack_rows(pool, data, 64, 2)
    cnn_desc, cnn_data, cnn_x, _ = models.cnn_small()
    with pytest.raises(ValueError, match=r"node 0 \(Conv\)"):
        models.stack_rows(cnn_desc, cnn_data, cnn_x.size, 2)
    with pytest.raises(ValueError, match=r"node 0 \(Dense\) takes 64 inputs but follows a tensor of 32"):
        models.stack_rows(desc, data, 32, 2)
    bad = desc.copy()
    bad[3, 2] = 128
    with pytest.raises(ValueError, match=r"node 3 \(Dense\) takes 128 inputs but follows a tensor of 64"):
        models.stack_rows(bad, data, 64, 2)
    tdesc, tdata, txs = token_mlp()
    with pytest.raises(ValueError, match=r"node 0 \(MatMul\) takes a \[8\]\[32\] matrix but follows a tensor of 128"):
        models.stack_rows(tdesc, tdata, 128, 2)
    bad = tdesc.copy()
    bad[3, 1] = 4
    with pytest.raises(ValueError, match=r"node 3 \(MatMul\) takes a \[4\]\[64\] matrix but follows a tensor of 512"):
        models.stack_rows(bad, tdata, txs.shape[1], 2)
    bad = desc.copy()
    bad[2, 0] = 9
    with pytest.raises(ValueError, match=r"node 2 has an unknown kind \(kind 9\)"):
        models.stack_rows(bad, data, 64, 2)


def test_pad_rows_copies_the_last_input():
    xs = np.arange(12, dtype=np.int64).reshape(3, 4)
    assert np.array_equal(models.pad_rows(xs, 4).reshape(4, 4), np.concatenate([xs, xs[2:]]))
    assert np.array_equal(models.pad_rows(xs, 8).reshape(8, 4)[3:], np.repeat(xs[2:], 5, axis=0))
    assert np.array_equal(models.pad_rows(xs[:1], 1), xs[0])
    for bad in (np.zeros((0, 4)), np.zeros((5, 4)), np.zeros(4)):
        with pytest.raises(ValueError, match="pad_rows"):
            models.pad_rows(bad, 4)


@pytest.mark.parametrize("rows", [1, 2, 3, 8, 5])
@pytest.mark.parametrize("name", list(MODELS))
def test_each_row_is_the_base_output(name, rows):
    """R = 1, 2 and 8, and rows = 3 and 5, whose last R - rows rows are copies of the last input"""
    desc, data, xs = MODELS[name]()
    sdesc, sdata, slen, R = models.stack_rows(desc, data, xs.shape[1], rows)
    group = xs[:rows]
    x = models.pad_rows(group, R)
    assert x.size == slen
    y = M.model_output(sdesc, sdata, x).reshape(R, -1)
    base = np.stack([M.model_output(desc, data, v) for v in group])
    assert y.shape[1] == base.shape[1]
    assert np.array_equal(y[:rows], base)
    assert np.array_equal(y[rows:], np.repeat(base[-1:], R - rows, axis=0))


@pytest.mark.parametrize("name,rows", [("mlp_2x64", 1), ("mlp_2x64", 8), ("mlp_2x64", 3), ("iris_calibrated", 30), ("iris_calibrated", 1)])
def test_checker_proves_stacked_and_verifier_checks_output(name, rows):
    """the checker proves the stacked model; the verifier accepts the true [R][N] output and rejects it with one element of one row
    changed"""
    desc, data, xs = MODELS[name]()
    sdesc, sdata, _, R = models.stack_rows(desc, data, xs.shape[1], rows)
    x = models.pad_rows(xs[:rows], R)
    y = M.model_output(sdesc, sdata, x)
    assert M.model_verify_output(sdesc, sdata, x, y) is None
    n = y.size // R
    bad = y.copy()
    bad[(rows - 1) * n + 1] += 1
    assert M.model_verify_output(sdesc, sdata, x, bad) is not None
    assert O.model_prove_verify(sdesc, sdata, x) is None
