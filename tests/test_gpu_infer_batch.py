"""dph_zkml_infer_batch on the H100: the models' outputs for batches of distinct inputs on the int8 tensor cores, without proving.
Outputs are pinned word for word to the checker's inference (zk_run(...).back()) and to the prover's own outputs (prove_batch,
trace_output); failing inputs fail alone with prove_batch's status and message; the plan's refusals name the node.

The checker's inference of the larger models takes 0.1 s (Dense-4M) to 3 s (the covid model at 224x224) per input on the CPU, so in
their 300-input batches it checks a spread sample of inputs; every input of every batch of the smaller models is checked.  A
batch's first inputs are the smaller batches' inputs, and their outputs must agree."""
import ctypes as C
import os
import re
import threading
import time

import numpy as np
import pytest

import models
import onnx_import as I
import oracle_model_io as M
import oracle_py as O
from test_gpu_prove_batch import _mlp_desc
from test_onnx_calibration import AGREEMENT_FLOOR, GOLDEN, samples
from test_onnx_import import _int_forward

pytestmark = pytest.mark.gpu
SIZES = (1, 7, 300)                   # none of them fills the GEMM's 64-row tiles evenly
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _images(n, c_u, img, seed):
    """n distinct inputs in the padded [p2(c_u)][p2(img)][p2(img)] layout, real pixels in [-127, 127]"""
    c_p, n_p = 1 << (c_u - 1).bit_length(), 1 << (img - 1).bit_length()
    x = np.zeros((n, c_p, n_p, n_p), dtype=np.int64)
    x[:, :c_u, :img, :img] = np.random.Generator(np.random.PCG64(seed)).integers(-127, 128, size=(n, c_u, img, img))
    return x.reshape(n, -1)


def _vectors(n, size, seed):
    return np.random.Generator(np.random.PCG64(seed)).integers(-127, 128, size=(n, size)).astype(np.int64)


def _onnx(name, calibrated):
    path = os.path.join(GOLDEN, name + ".onnx")
    cal = samples(name)[0] if calibrated else None
    desc, data, _, md = I.import_onnx(path, cal)[:4]
    floats = np.random.Generator(np.random.PCG64(31)).uniform(-1, 1, size=(max(SIZES),) + md.input_shape).astype(np.float32)
    return desc, data, np.stack([md.quantize_input(f) for f in floats])


def _model(name):
    """(desc, data, [300, input_len] distinct seeded inputs)"""
    if name == "mlp_2x64":
        return _mlp_desc() + (_vectors(max(SIZES), 64, 5),)
    if name == "dense4m":
        return _mlp_desc(4, 1024, 1) + (_vectors(max(SIZES), 1024, 6),)
    if name == "cnn_small":
        return models.cnn_small(seed=3)[:2] + (_images(max(SIZES), 3, 16, 7),)
    if name == "cnn264k":
        return models.cnn(seed=1)[:2] + (_images(max(SIZES), 3, 32, 8),)
    if name == "covid4":
        return models.covid(seed=3, channels=(4, 4, 4, 4, 4), fc=8)[:2] + (_images(max(SIZES), 3, 224, 9),)
    if name == "token_mlp":             # MatMul plain (with bias), then TransposeB (without)
        desc, data, x = models.token_mlp(seed=11, tokens=8, d_model=32, d_hidden=64)
        return desc, data, _vectors(max(SIZES), x.size, 10)
    onnx, quant = name.rsplit("-", 1)
    return _onnx(onnx, quant == "cal")


SMALL = ["mlp_2x64", "cnn_small", "token_mlp", "mlp-iris-01-absmax", "mlp-iris-01-cal"]
LARGE = ["cnn264k", "dense4m", "covid4", "cnn-cifar-01-absmax", "cnn-cifar-01-cal"]
_CACHE = {}


def _cached(name):
    if name not in _CACHE:
        _CACHE[name] = _model(name)
    return _CACHE[name]


@pytest.mark.parametrize("name", SMALL + LARGE)
def test_infer_equals_checker(gpu, name):
    desc, data, xs = _cached(name)
    ctx = gpu.ModelContext(desc, data, xs.shape[1])
    try:
        prev = None
        for n in SIZES:
            _, out, status, errors = ctx.infer_batch(xs[:n])
            assert out.shape == (n, ctx.output_len)
            assert status.tolist() == [0] * n and errors == [None] * n, errors
            if prev is not None:
                assert np.array_equal(out[: prev.shape[0]], prev), "%s: a batch of %d disagrees with the smaller batch" % (name, n)
            prev = out
            check = range(n) if name in SMALL else sorted({0, n // 2, n - 1} if name == "covid4" else {0, min(1, n - 1), n // 2, n - 1})
            for j in check:
                assert np.array_equal(out[j], M.model_output(desc, data, xs[j])), "%s: input %d of %d differs from the checker" % (name, j, n)
    finally:
        ctx.free()


@pytest.mark.parametrize("name", SMALL + ["cnn264k", "dense4m"])
def test_infer_equals_the_prover(gpu, name):
    """for a few inputs: prove_batch's outputs, and trace_output after prove(x), equal infer_batch's"""
    desc, data, xs = _cached(name)
    xs = xs[:3]
    ctx = gpu.ModelContext(desc, data, xs.shape[1])
    try:
        _, out, status, _ = ctx.infer_batch(xs)
        assert (status == 0).all()
        _, _, pout, pstatus, _ = ctx.prove_batch(xs, 3)
        assert (pstatus == 0).all() and np.array_equal(pout, out)
        for j in range(len(xs)):
            ctx.prove(xs[j])
            assert np.array_equal(ctx.trace_output(), out[j]), "%s: input %d" % (name, j)
    finally:
        ctx.free()


def test_full_channel_covid_equals_run_inference(gpu):
    """the full-channel covid model (models.covid()): two inputs equal the per-input device path (run_inference + trace_output)"""
    desc, data, _, _ = models.covid(seed=1)
    xs = _images(2, 3, 224, 12)
    ctx = gpu.ModelContext(desc, data, xs.shape[1])
    try:
        _, out, status, errors = ctx.infer_batch(xs)
        assert status.tolist() == [0, 0], errors
        for j in range(2):
            ctx.run_inference(xs[j])
            assert np.array_equal(ctx.trace_output(), out[j]), "input %d" % j
    finally:
        ctx.free()


def _max_chunk():
    src = open(os.path.join(ROOT, "include", "deepprove_b200.h")).read()
    return int(re.search(r"#define DP_INFER_MAX_CHUNK (\d+)", src).group(1))


def test_chunk_boundary(gpu):
    """a batch of (chunk cap + 3) inputs crosses a chunk boundary; inputs on both sides of it equal the checker, and the whole batch
    equals the same inputs inferred in batches of 300"""
    desc, data, _ = _cached("cnn_small")
    cap = _max_chunk()
    xs = _images(cap + 3, 3, 16, 13)
    ctx = gpu.ModelContext(desc, data, xs.shape[1])
    try:
        _, out, status, _ = ctx.infer_batch(xs)
        assert (status == 0).all()
        for j in (0, 1, cap - 2, cap - 1, cap, cap + 1, cap + 2):
            assert np.array_equal(out[j], M.model_output(desc, data, xs[j])), "input %d" % j
        parts = np.concatenate([ctx.infer_batch(xs[k: k + 300])[1] for k in range(0, len(xs), 300)])
        assert np.array_equal(parts, out)
    finally:
        ctx.free()


def test_failing_inputs_fail_alone(gpu):
    """the 2x64 MLP with its first requant's input bound cut to 2^14: full-range inputs overflow it, inputs in [-1, 1] do not.  A mixed
    batch gets the same statuses and messages from infer_batch and prove_batch, and the passing inputs equal the checker; an input
    value of 200 fails alone with its own message"""
    desc, data = _mlp_desc()
    desc = desc.copy()
    desc[1, 4] = 14
    rng = np.random.Generator(np.random.PCG64(21))
    xs = np.stack([rng.integers(-1, 2, size=64) if j % 2 == 0 else rng.integers(-127, 128, size=64) for j in range(8)]).astype(np.int64)
    ctx = gpu.ModelContext(desc, data, 64)
    try:
        _, out, status, errors = ctx.infer_batch(xs)
        _, _, pout, pstatus, perrors = ctx.prove_batch(xs, 4)
        assert status.tolist() == pstatus.tolist() and errors == perrors
        failed = [j for j in range(8) if status[j] != 0]
        assert failed and len(failed) < 8 and any("requantisation" in errors[j] for j in failed), errors
        for j in range(8):
            if j in failed:
                with pytest.raises(RuntimeError):
                    M.model_output(desc, data, xs[j])
            else:
                assert np.array_equal(out[j], M.model_output(desc, data, xs[j])) and np.array_equal(out[j], pout[j]), "input %d" % j
        ok = [j for j in range(8) if j not in failed]
        bad = xs[ok[:3]].copy()
        bad[1, 5] = 200
        _, out2, status2, errors2 = ctx.infer_batch(bad)
        assert status2.tolist() == [0, gpu.DP_ERR_INVALID, 0] and errors2[0] is None and errors2[2] is None
        assert "outside [-128, 127]" in errors2[1]
        assert np.array_equal(out2[[0, 2]], out[[ok[0], ok[2]]])
    finally:
        ctx.free()


def _refused(gpu, desc, data, x, node):
    ctx = gpu.ModelContext(desc, data, x.size)
    try:
        with pytest.raises(gpu.DpError) as e:
            ctx.infer_batch(x[None])
        assert e.value.code == gpu.DP_ERR_INVALID and ("node %d " % node) in str(e.value), str(e.value)
        return ctx, str(e.value)
    except BaseException:
        ctx.free()
        raise


def test_plan_refusals(gpu):
    desc, data = _mlp_desc()
    x = _vectors(1, 64, 22)[0]
    # a weight of 300 (node 3: the second Dense); proving on the handle still matches the checker
    d = data.copy()
    d[64 * 64 + 64 + 5] = 300
    ctx, msg = _refused(gpu, desc, d, x, 3)
    try:
        assert "weight 300" in msg
        assert np.array_equal(ctx.prove(x), O.model_prove(desc, d, x)[0])
        assert np.array_equal(ctx.trace_output(), M.model_output(desc, d, x))
    finally:
        ctx.free()
    # a Dense fed by a wide tensor: the first Requant removed, so the second Dense reads the first one's int32 outputs through Relu
    ctx, msg = _refused(gpu, np.delete(desc, 1, axis=0), data, x, 2)
    ctx.free()
    assert "not 8-bit" in msg
    # a row over the int32 bound: a bias just under 2^31 beside non-zero weights
    d = data.copy()
    d[64 * 64] = (1 << 31) - 2
    ctx, msg = _refused(gpu, desc, d, x, 0)
    ctx.free()
    assert "exceed int32" in msg


def test_busy_pool_and_stored_trace(gpu):
    """a call while the handle's pool proves a batch is refused with DP_ERR_STATE; an infer call leaves the stored trace's output as it
    was; a null handle is refused"""
    desc, data, xs = _cached("cnn_small")
    ctx = gpu.ModelContext(desc, data, xs.shape[1])
    try:
        out = np.zeros(16, dtype=np.int64)
        st = np.zeros(1, dtype=np.int32)
        assert gpu.host().dph_zkml_infer_batch(None, xs[:1].ctypes.data_as(C.c_void_p), 1, out.ctypes.data_as(C.c_void_p),
                                               st.ctypes.data_as(C.c_void_p), None) == gpu.DP_ERR_INVALID
        assert b"null handle" in gpu.host().dph_last_error()
        ctx.run_inference(xs[0])
        y0 = ctx.trace_output()
        _, out, _, _ = ctx.infer_batch(xs[1:5])
        assert np.array_equal(ctx.trace_output(), y0) and not np.array_equal(out[0], y0)
        ctx.prove_batch(xs[:1], 1)                 # sizes the default stride, so the thread's call goes straight to the pool
        res = {}
        t = threading.Thread(target=lambda: res.update(r=ctx.prove_batch(np.repeat(xs[:6], 8, axis=0), 1)))
        t.start()
        time.sleep(0.5)
        with pytest.raises(gpu.DpError) as e:
            ctx.infer_batch(xs[:2])
        t.join()
        assert e.value.code == gpu.DP_ERR_STATE and "busy" in str(e.value)
        assert (res["r"][3] == 0).all()
        _, out2, status, _ = ctx.infer_batch(xs[1:5])
        assert (status == 0).all() and np.array_equal(out2, out)
    finally:
        ctx.free()


def test_infer_batch_float_cifar_accuracy(gpu):
    """infer_batch_float of the calibrated CIFAR model on the reference's 30 samples: the checker's outputs, and the argmax agreement
    with the float model that the CPU test measures"""
    name = "cnn-cifar-01"
    path, (xs, _) = os.path.join(GOLDEN, name + ".onnx"), samples(name)
    ctx = gpu.ModelContext.from_onnx(path, calibration=xs)
    try:
        desc, data, _, md, fm, q = I.import_onnx(path, xs)
        outputs, floats, status, errors = ctx.infer_batch_float(xs)
        assert status.tolist() == [0] * len(xs) and errors == [None] * len(xs)
        for j in (0, 11, 29):
            assert np.array_equal(outputs[j], M.model_output(desc, data, md.quantize_input(xs[j])))
        f = [np.argmax(fm.forward(x)) for x in xs]
        agree = sum(int(np.argmax(floats[j]) == f[j]) for j in range(len(xs)))
        cpu = sum(int(np.argmax(_int_forward(fm, q, md.input_scaling.quantize(x))) == f[j]) for j, x in enumerate(xs))
        assert agree == cpu >= AGREEMENT_FLOOR[name]["all"]
    finally:
        ctx.free()
