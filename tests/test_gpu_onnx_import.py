"""Imported ONNX models (tests/golden/onnx/) proved on the H100: ModelContext.from_onnx proofs are word for word the checker's, and
prove_batch_float returns for every float input the checker's integer output, its dequantised floats and a proof the restated
verifier accepts with that output."""
import os

import numpy as np
import pytest

import oracle_model_io as M
import oracle_py as O

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "onnx")
MODELS = ["mlp-iris-01", "cnn-cifar-01"]


def _inputs(ctx, n, seed):
    return np.random.default_rng(seed).uniform(-1, 1, size=(n,) + ctx.metadata.input_shape).astype(np.float32)


@pytest.mark.parametrize("name", MODELS)
def test_prove_matches_checker(gpu, name):
    ctx = gpu.ModelContext.from_onnx(os.path.join(GOLDEN, name + ".onnx"))
    import onnx_import
    desc, data = onnx_import.import_onnx(os.path.join(GOLDEN, name + ".onnx"))[:2]
    for x in _inputs(ctx, 2, 21):
        xq = ctx.metadata.quantize_input(x)
        got = ctx.prove(xq)
        exp, _ = O.model_prove(desc, data, xq)
        assert got.shape == exp.shape and np.array_equal(got, exp)
        assert np.array_equal(ctx.trace_output(), M.model_output(desc, data, xq))


@pytest.mark.parametrize("name", MODELS)
def test_prove_batch_float(gpu, name):
    path = os.path.join(GOLDEN, name + ".onnx")
    ctx = gpu.ModelContext.from_onnx(path)
    import onnx_import
    desc, data = onnx_import.import_onnx(path)[:2]
    xs = _inputs(ctx, 8, 31)
    proofs, outputs, floats, status, errors = ctx.prove_batch_float(xs, n_workers=4)
    md = ctx.metadata
    assert status.tolist() == [0] * 8 and errors == [None] * 8
    assert floats.shape == (8, md.output_len)
    for j, x in enumerate(xs):
        xq = md.quantize_input(x)
        assert np.array_equal(outputs[j], M.model_output(desc, data, xq))
        assert np.array_equal(floats[j], outputs[j, :md.output_len].astype(np.float32) * md.output_scaling.scale)
        exp, _ = O.model_prove(desc, data, xq)
        assert np.array_equal(proofs[j], exp)
        assert M.model_verify_output(desc, data, xq, outputs[j]) is None
    assert len({p.tobytes() for p in proofs}) == 8
