"""ONNX import (deep-prove_b200/onnx_import.py) on the CPU: the two float models the reference ships (tests/golden/onnx/) parse to
their graphs, their float forward matches torch, the quantised integer model the checker runs equals a plain unpadded numpy
inference, the checker proves both and the restated verifier accepts each proof with its output, and every unsupported graph is
refused with an error that names the op or the attribute.  Float inputs are drawn from a seeded generator in [-1, 1]."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import onnx_import as I
import oracle_model_io as M

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "onnx")
IRIS, CIFAR = os.path.join(GOLDEN, "mlp-iris-01.onnx"), os.path.join(GOLDEN, "cnn-cifar-01.onnx")
# argmax agreement of the quantised model with the float model over the 64 seeded inputs of test_argmax_agreement, measured on
# this importer; kept as floors so a change in the quantisation shows up
ARGMAX_FLOOR = {IRIS: 64, CIFAR: 6}


def _inputs(fm, n, seed):
    return np.random.default_rng(seed).uniform(-1, 1, size=(n,) + fm.input_shape).astype(np.float32)


def _requant(x, rq):
    """Requant::op (layers/requant.rs:455-481) on an int64 array"""
    rs, fp, fpm, bits = rq
    sh = rs + fp
    assert np.all(np.abs(x) <= 1 << bits), "a value is outside the requantisation table"
    u = ((1 << (sh - 1)) + x * fpm) >> sh
    return np.where(np.abs(u) >= I.Q_MAX, I.Q_MAX * np.sign(u), u)


def _int_forward(fm, qlayers, xq):
    """straightforward unpadded integer inference of the quantised layers"""
    x = np.asarray(xq, dtype=np.int64).reshape(fm.input_shape)
    for q in qlayers:
        if q.kind == "dense":
            x = q.w @ x.reshape(-1) + q.b
        elif q.kind == "conv":
            k = q.w.shape[2]
            h = x.shape[1] - k + 1
            win = np.lib.stride_tricks.sliding_window_view(x, (k, k), axis=(1, 2))[:, :h, :h]
            x = np.einsum("ihwab,oiab->ohw", win, q.w) + q.b[:, None, None]
        elif q.kind == "relu":
            x = np.maximum(x, 0)
        elif q.kind == "maxpool":
            c, h, w = x.shape
            x = x[:, :h // 2 * 2, :w // 2 * 2].reshape(c, h // 2, 2, w // 2, 2).max(axis=(2, 4))
        else:
            x = x.reshape(-1)
        if q.rq is not None:
            x = _requant(x, q.rq)
    return x.reshape(-1)


_CACHE = {}


def _imported(path):
    if path not in _CACHE:
        _CACHE[path] = I.import_onnx(path)
    return _CACHE[path]


def test_fixtures_parse_to_their_graphs():
    fm = _imported(IRIS)[4]
    assert fm.input_shape == (4,)
    assert fm.ops() == ["dense", "relu"] * 4
    assert [l[1].shape for l in fm.layers if l[0] == "dense"] == [(30, 4), (30, 30), (30, 30), (3, 30)]
    fm = _imported(CIFAR)[4]
    assert fm.input_shape == (3, 32, 32)
    assert fm.ops() == ["conv", "relu", "maxpool"] * 2 + ["flatten", "dense", "relu", "dense", "relu", "dense"]
    assert [l[1].shape for l in fm.layers if l[0] == "conv"] == [(6, 3, 5, 5), (16, 6, 5, 5)]
    assert [l[1].shape for l in fm.layers if l[0] == "dense"] == [(120, 400), (84, 120), (10, 84)]
    assert all(l[2].shape == (l[1].shape[0],) for l in fm.layers if len(l) == 3)


def test_padded_descriptors():
    desc, data, input_len, md = _imported(IRIS)[:4]
    assert input_len == 4 and md.padded_input_shape == (4,) and md.output_len == 3 and md.padded_output_len == 4
    assert desc[:, 0].tolist() == [I.models.DENSE, I.REQUANT, I.RELU] * 4
    assert [tuple(d[1:3]) for d in desc if d[0] == I.models.DENSE] == [(32, 4), (32, 32), (32, 32), (4, 32)]
    desc, data, input_len, md = _imported(CIFAR)[:4]
    assert input_len == 4 * 32 * 32 and md.output_len == 10 and md.padded_output_len == 16
    assert desc[-1, 0] == I.REQUANT              # the reference appends a requant after every dense layer, the last one too
    assert [tuple(d[1:3]) for d in desc if d[0] == I.models.DENSE] == [(128, 1024), (128, 128), (16, 128)]
    assert [d[:8].tolist() for d in desc if d[0] == I.models.CONV] == [[3, 8, 4, 32, 8, 6, 28, 28], [3, 16, 8, 16, 8, 16, 10, 10]]
    for d in desc[desc[:, 0] == I.REQUANT]:
        assert (d[1] + d[2]) % I.BIT_LEN == 0 and d[2] >= I.FIXED_POINT_SCALE and d[4] + d[2] <= 63


@pytest.mark.parametrize("path", [IRIS, CIFAR], ids=["iris", "cifar"])
def test_float_forward_matches_torch(path):
    fm = _imported(path)[4]
    for x in _inputs(fm, 4, 5):
        t = torch.from_numpy(x)[None]
        for l in fm.layers:
            if l[0] == "dense":
                t = F.linear(t, torch.from_numpy(l[1]), torch.from_numpy(l[2]))
            elif l[0] == "conv":
                t = F.conv2d(t, torch.from_numpy(l[1]), torch.from_numpy(l[2]))
            elif l[0] == "relu":
                t = F.relu(t)
            elif l[0] == "maxpool":
                t = F.max_pool2d(t, 2, 2)
            else:
                t = t.flatten(1)
        y = t.numpy().reshape(-1).astype(np.float64)
        np.testing.assert_allclose(fm.forward(x), y, rtol=1e-5, atol=1e-5 * np.abs(y).max())


@pytest.mark.parametrize("path", [IRIS, CIFAR], ids=["iris", "cifar"])
def test_checker_output_equals_unpadded_integer_inference(path):
    desc, data, _, md, fm, q = _imported(path)
    for x in _inputs(fm, 4, 7):
        xq = md.quantize_input(x)
        y = M.model_output(desc, data, xq)
        assert y.size == md.padded_output_len
        assert np.array_equal(y[:md.output_len], _int_forward(fm, q, md.input_scaling.quantize(x)))
        assert np.array_equal(md.dequantize_output(y), y[:md.output_len].astype(np.float32) * md.output_scaling.scale)


@pytest.mark.parametrize("path", [IRIS, CIFAR], ids=["iris", "cifar"])
def test_argmax_agreement(path):
    """how often the quantised model's argmax equals the float model's (zkml/src/bin/bench.rs:454-464), over 64 seeded inputs"""
    _, _, _, md, fm, q = _imported(path)
    xs = _inputs(fm, 64, 11)
    agree = sum(int(np.argmax(_int_forward(fm, q, md.input_scaling.quantize(x))) == np.argmax(fm.forward(x))) for x in xs)
    print("argmax agreement %s: %d / 64" % (os.path.basename(path), agree))
    assert agree >= ARGMAX_FLOOR[path]


@pytest.mark.parametrize("path", [IRIS, CIFAR], ids=["iris", "cifar"])
def test_checker_proves_and_verifier_accepts(path):
    desc, data, _, md, fm, _ = _imported(path)
    xq = md.quantize_input(_inputs(fm, 1, 13)[0])
    y = M.model_output(desc, data, xq)
    assert M.model_verify_output(desc, data, xq, y) is None
    bad = y.copy()
    bad[md.output_len - 1] += 1
    assert M.model_verify_output(desc, data, xq, bad) is not None


def test_quantize_input_rule():
    md = _imported(CIFAR)[3]
    x = np.zeros((3, 32, 32), dtype=np.float32)
    x[0, 0, :4] = [1.0, -1.0, 0.5, 1.0 / 254]      # 1/254 / (2/254) = 0.5: rounds away from zero
    q = md.quantize_input(x).reshape(4, 32, 32)
    assert q[0, 0, :4].tolist() == [127, -127, 64, 1] and q.sum() == 127 - 127 + 64 + 1
    assert md.quantize_input(np.stack([x, x])).shape == (2, 4096)
    with pytest.raises(ValueError, match=r"\[-1, 1\]"):
        md.quantize_input(x + 1.5)
    with pytest.raises(ValueError, match="shape"):
        md.quantize_input(np.zeros((3, 16, 16), dtype=np.float32))


def test_requant_from_multiplier():
    """m = 0.75 * 2^-7: right shift 7, fp_scale 25 (7 + 25 = 32) and a multiplier of about 0.75 * 2^25 -- log2 and powf in f32 lose
    the last bits, as they do in the reference; m = 0.75 * 2^-9: 9 + 31 = 40"""
    rs, fp, fpm = I.requant_from_multiplier(np.float32(0.75 / 128), 20)
    assert (rs, fp) == (7, 25) and abs(fpm - (3 << 23)) <= (3 << 23) * 1e-6
    rs, fp, fpm = I.requant_from_multiplier(np.float32(0.75 / 512), 20)
    assert (rs, fp) == (9, 31) and abs(fpm - (3 << 29)) <= (3 << 29) * 1e-6
    with pytest.raises(ValueError, match="exceeds 63"):
        I.requant_from_multiplier(np.float32(0.75 / 512), 33)


# ---- refusals: tiny models written with the same protobuf wire encoding --------------------------------------------------

def _key(f, t):
    return _vint((f << 3) | t)


def _vint(v):
    v &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def _ld(f, b):
    b = b.encode() if isinstance(b, str) else b
    return _key(f, 2) + _vint(len(b)) + b


def _vi(f, v):
    return _key(f, 0) + _vint(v)


def _attr_ints(name, vals):
    return _ld(1, name) + _ld(8, b"".join(_vint(v) for v in vals))          # packed


def _attr_int(name, v):
    return _ld(1, name) + _vi(3, v)


def _tensor(name, a):
    a = np.asarray(a, dtype=np.float32)
    return b"".join(_vi(1, d) for d in a.shape) + _vi(2, 1) + _ld(8, name) + _ld(9, a.astype("<f4").tobytes())


def _node(op, ins, outs, attrs=(), name=""):
    return b"".join(_ld(1, i) for i in ins) + b"".join(_ld(2, o) for o in outs) + _ld(3, name) + _ld(4, op) + b"".join(_ld(5, a) for a in attrs)


def _value_info(name, dims):
    shape = b"".join(_ld(1, _vi(1, d)) for d in dims)
    return _ld(1, name) + _ld(2, _ld(1, _vi(1, 1) + _ld(2, shape)))


def _model(nodes, inits, in_dims, out="y"):
    g = b"".join(_ld(1, n) for n in nodes) + b"".join(_ld(5, t) for t in inits)
    g += _ld(11, _value_info("x", in_dims)) + _ld(12, _value_info(out, [1]))
    return _ld(7, g)


def _conv_model(attrs, name="conv0"):
    rng = np.random.default_rng(0)
    w, b = rng.uniform(-1, 1, (2, 1, 3, 3)), rng.uniform(-1, 1, 2)
    wd, bd = rng.uniform(-1, 1, (4, 2 * 6 * 6)), rng.uniform(-1, 1, 4)
    nodes = [_node("Conv", ["x", "w", "b"], ["c"], attrs, name), _node("Flatten", ["c"], ["f"], [_attr_int("axis", 1)]),
             _node("Gemm", ["f", "wd", "bd"], ["y"], [_attr_int("transB", 1)])]
    return _model(nodes, [_tensor("w", w), _tensor("b", b), _tensor("wd", wd), _tensor("bd", bd)], [1, 1, 8, 8])


def test_tiny_encoded_model_imports():
    desc, data, input_len, md, fm, q = I.import_onnx(_conv_model([_attr_ints("pads", [0, 0, 0, 0]), _attr_ints("strides", [1, 1])]))
    assert fm.ops() == ["conv", "flatten", "dense"] and input_len == 64 and md.output_len == 4
    x = _inputs(fm, 1, 3)[0]
    y = M.model_output(desc, data, md.quantize_input(x))
    assert np.array_equal(y[:4], _int_forward(fm, q, md.input_scaling.quantize(x)))


@pytest.mark.parametrize("attr,match", [(_attr_ints("pads", [1, 1, 1, 1]), "pads"), (_attr_ints("strides", [2, 2]), "strides"),
                                        (_attr_ints("dilations", [2, 2]), "dilations"), (_attr_int("group", 2), "group")],
                         ids=["pads", "strides", "dilations", "group"])
def test_conv_attribute_refused(attr, match):
    with pytest.raises(ValueError, match=r"Conv node 'conv0'.*%s" % match):
        I.import_onnx(_conv_model([attr]))


def test_sigmoid_refused():
    w, b = np.ones((4, 4)), np.zeros(4)
    m = _model([_node("Gemm", ["x", "w", "b"], ["h"], [_attr_int("transB", 1)]), _node("Sigmoid", ["h"], ["y"], name="sig")],
               [_tensor("w", w), _tensor("b", b)], [1, 4])
    with pytest.raises(ValueError, match=r"Sigmoid node 'sig'.*unsupported op 'Sigmoid'"):
        I.import_onnx(m)


def test_maxpool_other_than_2x2_stride_2_refused():
    rng = np.random.default_rng(0)
    nodes = [_node("MaxPool", ["x"], ["p"], [_attr_ints("kernel_shape", [3, 3]), _attr_ints("strides", [3, 3])], "pool0"),
             _node("Flatten", ["p"], ["f"]), _node("Gemm", ["f", "wd", "bd"], ["y"], [_attr_int("transB", 1)])]
    m = _model(nodes, [_tensor("wd", rng.uniform(-1, 1, (4, 4))), _tensor("bd", np.zeros(4))], [1, 1, 6, 6])
    with pytest.raises(ValueError, match=r"MaxPool node 'pool0'.*2x2"):
        I.import_onnx(m)


def test_non_chain_refused():
    w, b = np.ones((4, 4)), np.zeros(4)
    nodes = [_node("Gemm", ["x", "w", "b"], ["h"], [_attr_int("transB", 1)], "g0"), _node("Relu", ["h"], ["r"], name="r0"),
             _node("Gemm", ["h", "w", "b"], ["y"], [_attr_int("transB", 1)], "g1")]     # g1 reads g0's output, skipping r0
    with pytest.raises(ValueError, match=r"Gemm node 'g1'.*single chain"):
        I.import_onnx(_model(nodes, [_tensor("w", w), _tensor("b", b)], [1, 4]))


def test_gemm_without_transb_and_matmul_are_dense():
    """Gemm with transB = 0 and a bias-less MatMul both hold their matrix as [in, out]: the imported dense layer is its transpose"""
    rng = np.random.default_rng(2)
    w1, b1, w2 = rng.uniform(-1, 1, (4, 8)), rng.uniform(-1, 1, 8), rng.uniform(-1, 1, (8, 4))
    nodes = [_node("Gemm", ["x", "w1", "b1"], ["h"]), _node("Relu", ["h"], ["r"]), _node("MatMul", ["r", "w2"], ["y"])]
    fm = I.import_onnx(_model(nodes, [_tensor("w1", w1), _tensor("b1", b1), _tensor("w2", w2)], [1, 4]))[4]
    x = _inputs(fm, 1, 4)[0].astype(np.float64)
    w1, b1, w2 = (a.astype(np.float32).astype(np.float64) for a in (w1, b1, w2))
    np.testing.assert_allclose(fm.forward(x), np.maximum(x @ w1 + b1, 0) @ w2, rtol=1e-6)
