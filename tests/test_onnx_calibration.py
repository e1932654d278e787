"""Calibrated ONNX import (onnx_import.observe / import_onnx(path, calibration)) on the CPU, with the reference's own samples
(tests/golden/onnx/*-inputs.npz, made by make_onnx_inputs.py): the calibrated scalings and requants follow the InferenceObserver
rule, an import without calibration is unchanged, the checker runs and proves the calibrated models, the quantised models agree
with the float ones far more often than under AbsoluteMax, and bad calibration sets are refused."""
import hashlib
import os

import numpy as np
import pytest

import onnx_import as I
import oracle_model_io as M
from test_onnx_import import _attr_int, _int_forward, _model, _node, _tensor

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "onnx")
MODELS = ["mlp-iris-01", "cnn-cifar-01"]
# argmax agreement of the quantised model with the float model on the reference's 30 samples, measured on this importer and kept as
# floors: calibrated on all 30 and evaluated on all 30, calibrated on 0-14 and evaluated on 15-29, and AbsoluteMax on all 30
AGREEMENT_FLOOR = {"mlp-iris-01": {"all": 29, "held_out": 14, "absmax": 28},
                   "cnn-cifar-01": {"all": 27, "held_out": 14, "absmax": 12}}
# SHA-256 of the uncalibrated (AbsoluteMax) import's descriptor and data, as little-endian int64, from before calibration existed
UNCALIBRATED_SHA256 = {"mlp-iris-01": "478bdfd908e845105d1d65534f78da882637e1539d5b2d4ad59da1fcaaf4bc24",
                       "cnn-cifar-01": "396218e94467012e8e04426ccd39a2a6559b353e96c47e0eec5acbaef6eeb12f"}


def samples(name):
    """(inputs float32 [30, *input shape], labels int64 [30])"""
    f = np.load(os.path.join(GOLDEN, name + "-inputs.npz"))
    return f["inputs"], f["labels"]


_CACHE = {}


def calibrated(name):
    """import_onnx calibrated on all 30 samples"""
    if name not in _CACHE:
        _CACHE[name] = I.import_onnx(os.path.join(GOLDEN, name + ".onnx"), samples(name)[0])
    return _CACHE[name]


@pytest.mark.parametrize("name", MODELS)
def test_scalings_follow_the_observer_rule(name):
    """input scaling from the samples' absolute maximum; each Dense / Conv output scaling from the absolute maximum of that layer's
    own float output over the samples (before its Relu), rounded to f32; each requant from (input, weight, output) scalings"""
    xs = samples(name)[0]
    _, _, _, md, fm, q = calibrated(name)
    assert md.input_scaling.scale == np.float32(2) * np.float32(np.abs(xs).max()) / np.float32(254)
    outs = [list(fm.outputs(x)) for x in xs]
    sf = md.input_scaling
    for i, (l, ql) in enumerate(zip(fm.layers, q)):
        if l[0] not in ("dense", "conv"):
            assert ql.rq is None and ql.out_sf is None
            continue
        a = np.float32(max(np.abs(o[i]).max() for o in outs))
        assert ql.out_sf.scale == np.float32(2) * a / np.float32(254) and ql.out_sf.domain == (I.Q_MIN, I.Q_MAX)
        w_sf = I.ScalingFactor.from_absolute_max(max(np.abs(l[1]).max(), np.abs(l[2]).max()))
        assert ql.rq == I.requant_from_multiplier(sf.scale * w_sf.scale / ql.out_sf.scale, ql.rq[3]) + (ql.rq[3],)
        assert np.array_equal(ql.w, w_sf.quantize(l[1]))
        sf = ql.out_sf
    assert md.output_scaling is sf


@pytest.mark.parametrize("name", MODELS)
def test_without_calibration_the_import_is_unchanged(name):
    desc, data, input_len, md, fm, q = I.import_onnx(os.path.join(GOLDEN, name + ".onnx"))
    h = hashlib.sha256(np.ascontiguousarray(desc, dtype="<i8").tobytes() + np.ascontiguousarray(data, dtype="<i8").tobytes())
    assert h.hexdigest() == UNCALIBRATED_SHA256[name]
    default = I.ScalingFactor.default().scale
    assert md.input_scaling.scale == default and md.output_scaling.scale == default
    assert all(ql.out_sf.scale == default for ql in q if ql.rq is not None)


@pytest.mark.parametrize("name", MODELS)
def test_calibrated_descriptor_fits_the_prover(name):
    """the requants of a calibrated model stay inside what the prover takes: shifts in whole bytes, at most 63 bits before the
    shift, and at most 8 lookup tables (dp_wit_begin): relu, range, and one clamping table per distinct clamping size
    (intermediate bits + ceil log2 of the multiplier - shift, layers/requant.rs:470-473)"""
    desc = calibrated(name)[0]
    rq = desc[desc[:, 0] == I.REQUANT]
    assert np.all((rq[:, 1] + rq[:, 2]) % I.BIT_LEN == 0) and np.all(rq[:, 4] + rq[:, 2] <= 63)
    clamping = sorted({int(b) + int(f - 1).bit_length() - int(s + p) for s, p, f, b in rq[:, 1:5]})
    print("%s: clamping tables of %s bits" % (name, clamping))
    assert 2 + len(clamping) <= 8


@pytest.mark.parametrize("name", MODELS)
def test_checker_output_equals_unpadded_integer_inference(name):
    desc, data, _, md, fm, q = calibrated(name)
    for x in samples(name)[0]:
        y = M.model_output(desc, data, md.quantize_input(x))
        assert np.array_equal(y[:md.output_len], _int_forward(fm, q, md.input_scaling.quantize(x)))


@pytest.mark.parametrize("name", MODELS)
def test_checker_proves_and_verifier_accepts(name):
    desc, data, _, md, fm, _ = calibrated(name)
    xq = md.quantize_input(samples(name)[0][3])
    y = M.model_output(desc, data, xq)
    assert M.model_verify_output(desc, data, xq, y) is None
    bad = y.copy()
    bad[md.output_len - 1] += 1
    assert M.model_verify_output(desc, data, xq, bad) is not None


def _agreement(fm, md, q, xs, labels):
    """(argmax agreement of quantised and float model, float accuracy, quantised accuracy) over xs"""
    f = np.array([np.argmax(fm.forward(x)) for x in xs])
    z = np.array([np.argmax(_int_forward(fm, q, md.input_scaling.quantize(x))) for x in xs])
    return int((f == z).sum()), int((f == labels).sum()), int((z == labels).sum())


@pytest.mark.parametrize("name", MODELS)
def test_argmax_agreement(name):
    """zkml/src/bin/bench.rs:454-464 compares the quantised and float argmax; the labels give each model's accuracy"""
    xs, labels = samples(name)
    path = os.path.join(GOLDEN, name + ".onnx")
    arms = {"all": (I.import_onnx(path, xs), slice(0, 30)), "held_out": (I.import_onnx(path, xs[:15]), slice(15, 30)),
            "absmax": (I.import_onnx(path), slice(0, 30))}
    for arm, (imp, ev) in arms.items():
        _, _, _, md, fm, q = imp
        agree, acc_f, acc_q = _agreement(fm, md, q, xs[ev], labels[ev])
        n = len(labels[ev])
        print("%s %s: argmax agreement %d / %d; accuracy float %d / %d, quantised %d / %d" % (name, arm, agree, n, acc_f, n, acc_q, n))
        assert agree >= AGREEMENT_FLOOR[name][arm]


def test_empty_calibration_refused():
    with pytest.raises(ValueError, match="no samples"):
        I.import_onnx(os.path.join(GOLDEN, "mlp-iris-01.onnx"), np.zeros((0, 4), np.float32))


@pytest.mark.parametrize("shape", [(30, 5), (4,), (30, 2, 2)], ids=["width", "no-batch", "rank"])
def test_calibration_shape_refused(shape):
    with pytest.raises(ValueError, match=r"shape \[n, 4\]"):
        I.import_onnx(os.path.join(GOLDEN, "mlp-iris-01.onnx"), np.zeros(shape, np.float32) + 0.5)


@pytest.mark.parametrize("bad", [1.5, -1.01, np.nan])
def test_calibration_values_outside_unit_range_refused(bad):
    xs = samples("mlp-iris-01")[0].copy()
    xs[7, 2] = bad
    with pytest.raises(ValueError, match=r"\[-1, 1\]"):
        I.import_onnx(os.path.join(GOLDEN, "mlp-iris-01.onnx"), xs)


def test_zero_node_output_refused():
    """a dense layer whose observed output is zero on every sample would get a zero scaling factor"""
    rng = np.random.default_rng(1)
    nodes = [_node("Gemm", ["x", "w1", "b1"], ["h"], [_attr_int("transB", 1)], "g0"), _node("Relu", ["h"], ["r"]),
             _node("Gemm", ["r", "w2", "b2"], ["y"], [_attr_int("transB", 1)], "g1")]
    m = _model(nodes, [_tensor("w1", rng.uniform(-1, 1, (4, 4))), _tensor("b1", np.zeros(4)), _tensor("w2", np.zeros((4, 4))),
                       _tensor("b2", np.zeros(4))], [1, 4])
    xs = rng.uniform(-1, 1, (5, 4)).astype(np.float32)
    with pytest.raises(ValueError, match=r"output of layer 2 \(dense\) is zero on every sample"):
        I.import_onnx(m, xs)
    with pytest.raises(ValueError, match="the input is zero on every sample"):
        I.import_onnx(m, np.zeros_like(xs))


def test_zero_relu_output_is_not_refused():
    """a Relu keeps its input's scaling, so its own all-zero output (here: the first dense layer is negative on every sample) does
    not matter, as in the reference, where the Activation's observed scaling is discarded"""
    nodes = [_node("Gemm", ["x", "w1", "b1"], ["h"], [_attr_int("transB", 1)]), _node("Relu", ["h"], ["r"]),
             _node("Gemm", ["r", "w2", "b2"], ["y"], [_attr_int("transB", 1)])]
    m = _model(nodes, [_tensor("w1", np.zeros((4, 4))), _tensor("b1", -np.ones(4)), _tensor("w2", np.ones((4, 4))),
                       _tensor("b2", np.full(4, 0.5))], [1, 4])
    q = I.import_onnx(m, np.full((3, 4), 0.25, np.float32))[5]
    assert [ql.out_sf.scale for ql in q if ql.rq is not None] == [np.float32(2) / 254, np.float32(1) / 254]
