"""Calibrated ONNX models (ModelContext.from_onnx(path, calibration)) proved on the H100 with the reference's shipped samples: device
proofs are word for word the checker's, and prove_batch_float on all 30 CIFAR samples returns the checker's outputs, proofs the
restated verifier accepts, and dequantised outputs with the argmax agreement the CPU test measures."""
import os

import numpy as np
import pytest

import onnx_import as I
import oracle_model_io as M
import oracle_py as O
from test_onnx_calibration import AGREEMENT_FLOOR, GOLDEN, MODELS, samples
from test_onnx_import import _int_forward

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", MODELS)
def test_prove_matches_checker(gpu, name):
    path, xs = os.path.join(GOLDEN, name + ".onnx"), samples(name)[0]
    ctx = gpu.ModelContext.from_onnx(path, calibration=xs)
    desc, data = I.import_onnx(path, xs)[:2]
    for x in xs[[0, 17]]:
        xq = ctx.metadata.quantize_input(x)
        got = ctx.prove(xq)
        exp, _ = O.model_prove(desc, data, xq)
        assert got.shape == exp.shape and np.array_equal(got, exp)
        assert np.array_equal(ctx.trace_output(), M.model_output(desc, data, xq))


def test_prove_batch_float_cifar(gpu):
    name = "cnn-cifar-01"
    path, (xs, _) = os.path.join(GOLDEN, name + ".onnx"), samples(name)
    ctx = gpu.ModelContext.from_onnx(path, calibration=xs)
    desc, data, _, md, fm, q = I.import_onnx(path, xs)
    proofs, outputs, floats, status, errors = ctx.prove_batch_float(xs, n_workers=8)
    assert status.tolist() == [0] * len(xs) and errors == [None] * len(xs)
    for j, x in enumerate(xs):
        xq = md.quantize_input(x)
        assert np.array_equal(outputs[j], M.model_output(desc, data, xq))
        exp, _ = O.model_prove(desc, data, xq)
        assert np.array_equal(proofs[j], exp)
        assert M.model_verify_output(desc, data, xq, outputs[j]) is None
    f = [np.argmax(fm.forward(x)) for x in xs]
    agree = sum(int(np.argmax(floats[j]) == f[j]) for j in range(len(xs)))
    cpu = sum(int(np.argmax(_int_forward(fm, q, md.input_scaling.quantize(x))) == f[j]) for j, x in enumerate(xs))
    print("%s calibrated, device outputs: argmax agreement %d / %d" % (name, agree, len(xs)))
    assert agree == cpu >= AGREEMENT_FLOOR[name]["all"]
