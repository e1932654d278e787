"""dph_zkml_prove_batch on the H100: n distinct inputs proved end to end on the handle's worker pool, each returning its proof and
the model's output.  Every proof is pinned word for word to the checker's proof of the same input, every output to the checker's
inference, and the restated verifier accepts each (input, device output) pair.  One input that the quantised tables refuse fails
alone."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

import models
import oracle_model_io as M
import oracle_py as O

pytestmark = pytest.mark.gpu
N_INPUTS, N_WORKERS = 6, 4


def _mlp_desc(n_layers=2, width=64, seed=5):
    """the 2x64 synthetic MLP as a layer descriptor (what ZkmlContext builds from it)"""
    w, b, rq = O.synthetic_mlp(n_layers, width, seed)
    desc = np.zeros((3 * n_layers, 9), dtype=np.int64)
    desc[0::3, 1:3] = width
    desc[1::3, 0], desc[1::3, 1:5] = 1, rq
    desc[2::3, 0] = 2
    return desc, np.concatenate([w.reshape(n_layers, -1), b.reshape(n_layers, -1)], axis=1).reshape(-1)


def _model(name):
    """(desc, data, [N_INPUTS, input_len] distinct seeded inputs)"""
    if name == "mlp_2x64":
        desc, data = _mlp_desc()
        xs = [O.synthetic_input(64, 6 + j) for j in range(N_INPUTS)]
    elif name == "cnn_small":
        desc, data, _, _ = models.cnn_small(seed=3)
        xs = [models.cnn_small(seed=100 + j)[2] for j in range(N_INPUTS)]     # the padded input layout, drawn from other seeds
    else:
        desc, data, x = models.token_mlp(seed=11, tokens=8, d_model=32, d_hidden=64)
        rng = np.random.Generator(np.random.PCG64(7))
        xs = [rng.integers(-127, 128, size=x.size).astype(np.int64) for _ in range(N_INPUTS)]
    return desc, data, np.stack(xs).astype(np.int64)


_EXPECTED = {}


def _expected(name, hasher, desc, data, xs):
    """the checker's proof and output of every input (cached per model and hasher)"""
    key = (name, hasher)
    if key not in _EXPECTED:
        _EXPECTED[key] = [(O.model_prove(desc, data, x)[0], M.model_output(desc, data, x)) for x in xs]
    return _EXPECTED[key]


@pytest.fixture()
def wait_mode(gpu, request):
    before = gpu.lib().dp_get_wait_mode()
    gpu.set_wait_mode(request.param)
    yield request.param
    gpu.set_wait_mode(before)


def _check_batch(gpu, name, hasher):
    desc, data, xs = _model(name)
    exp = _expected(name, hasher, desc, data, xs)
    ctx = gpu.ModelContext(desc, data, xs.shape[1])
    try:
        _, proofs, outputs, status, errors = ctx.prove_batch(xs, N_WORKERS, stride=exp[0][0].size + 64)
        assert (status == 0).all() and errors == [None] * N_INPUTS, errors
        assert outputs.shape == (N_INPUTS, ctx.output_len)
        for j, (p, y) in enumerate(exp):
            assert proofs[j].size == p.size and (proofs[j] == p).all(), "%s: proof of input %d differs from the checker's" % (name, j)
            assert (outputs[j] == y).all(), "%s: output of input %d differs from the checker's inference" % (name, j)
        assert len({p.tobytes() for p in proofs}) == N_INPUTS, "%s: two distinct inputs gave the same proof" % name
        for j in range(N_INPUTS):          # the single-proof path on the same input agrees, proof and stored-trace output
            assert (ctx.prove(xs[j]) == proofs[j]).all(), "%s: dph_zkml_prove differs on input %d" % (name, j)
            assert (ctx.trace_output() == outputs[j]).all(), "%s: trace_output differs on input %d" % (name, j)
    finally:
        ctx.free()
    return xs, outputs, desc, data


@pytest.mark.parametrize("wait_mode", [0, 1], indirect=True, ids=["spin", "blocking"])
@pytest.mark.parametrize("name", ["mlp_2x64", "cnn_small", "token_mlp"])
def test_batch_equals_checker(gpu, wait_mode, name):
    xs, outputs, desc, data = _check_batch(gpu, name, 0)
    if wait_mode == 0:                     # the public IO: the verifier accepts each input with the output the device returned
        for j in range(N_INPUTS):
            assert M.model_verify_output(desc, data, xs[j], outputs[j]) is None, "%s: input %d" % (name, j)


@pytest.mark.parametrize("wait_mode", [1], indirect=True, ids=["blocking"])
def test_batch_equals_checker_blake(gpu, wait_mode):
    O.set_hash_mode(1); gpu.set_hasher(1)
    try:
        xs, outputs, desc, data = _check_batch(gpu, "token_mlp", 1)
        assert M.model_verify_output(desc, data, xs[0], outputs[0]) is None
    finally:
        O.set_hash_mode(0); gpu.set_hasher(0)


@pytest.mark.parametrize("wait_mode", [0, 1], indirect=True, ids=["spin", "blocking"])
def test_failing_input_fails_alone(gpu, wait_mode):
    """input 2, scaled far outside the quantised range, overflows the first requantisation: only its job fails, the others still
    equal the checker, and the handle proves a normal batch afterwards"""
    desc, data, xs = _model("mlp_2x64")
    exp = _expected("mlp_2x64", 0, desc, data, xs)
    bad = xs.copy()
    bad[2] *= 4096
    with pytest.raises(RuntimeError, match="requantisation"):
        M.model_output(desc, data, bad[2])
    ctx = gpu.ModelContext(desc, data, xs.shape[1])
    try:
        stride = exp[0][0].size + 64
        _, proofs, outputs, status, errors = ctx.prove_batch(bad, N_WORKERS, stride=stride)
        assert [j for j in range(N_INPUTS) if status[j] != 0] == [2]
        assert proofs[2].size == 0 and "requantisation" in errors[2]
        for j, (p, y) in enumerate(exp):
            if j != 2:
                assert errors[j] is None and (proofs[j] == p).all() and (outputs[j] == y).all(), "input %d" % j
        _, proofs, outputs, status, errors = ctx.prove_batch(xs, N_WORKERS, stride=stride)
        assert (status == 0).all() and errors == [None] * N_INPUTS
        for j, (p, y) in enumerate(exp):
            assert (proofs[j] == p).all() and (outputs[j] == y).all(), "input %d after the failed batch" % j
    finally:
        ctx.free()


def test_batch_refusals(gpu):
    """call-level refusals on a real handle: a stride too small for a proof, an output buffer too small for trace_output, a trace
    output before any trace, and a batch call while the handle's pool is busy with another"""
    desc, data, xs = _model("cnn_small")
    ctx = gpu.ModelContext(desc, data, xs.shape[1])
    H = gpu.host()
    try:
        assert ctx.output_len == 16
        with pytest.raises(gpu.DpError) as e:
            ctx.trace_output()
        assert e.value.code == gpu.DP_ERR_STATE
        with pytest.raises(gpu.DpError, match="longer than the stride"):
            ctx.prove_batch(xs[:2], 2, stride=16)
        ctx.run_inference(xs[0])
        small, n = np.zeros(8, dtype=np.int64), C.c_uint64()
        assert H.dph_zkml_trace_output(ctx.h, small.ctypes.data_as(C.c_void_p), small.size, C.byref(n)) == gpu.DP_ERR_INVALID
        assert n.value == 16 and b"too small" in H.dph_last_error()
        # busy pool: a long batch on one worker in another thread (ctypes releases the GIL), then a second call on the same handle
        ctx.prove_batch(xs[:1], 1)         # sizes the default stride, so the thread's call goes straight to the pool
        res = {}
        t = threading.Thread(target=lambda: res.update(r=ctx.prove_batch(np.repeat(xs, 8, axis=0), 1)))
        t.start()
        time.sleep(0.5)
        with pytest.raises(gpu.DpError) as e:
            ctx.prove_batch(xs[:1], 1)
        t.join()
        assert e.value.code == gpu.DP_ERR_STATE and "busy" in str(e.value)
        assert (res["r"][3] == 0).all()
    finally:
        ctx.free()
