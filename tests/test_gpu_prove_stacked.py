"""StackedContext.prove_stacked on the H100: many inputs of an MLP in one proof, as the rows of the reference's Input x Weight MatMul.
Every stacked proof is pinned word for word to the checker's proof of the same padded input matrix, each group's output matrix is
accepted by the restated verifier, and each input's output equals what prove_batch and infer_batch return for it.  An input that
screening refuses is left out of its group with infer_batch's message, and the rest of the group is still proved."""
import os
import threading
import time

import numpy as np
import pytest

import models
import oracle_model_io as M
import oracle_py as O
from test_gpu_prove_batch import _mlp_desc
from test_stack_rows import GOLDEN, MODELS, iris, samples

pytestmark = pytest.mark.gpu
N_WORKERS = 4


@pytest.fixture()
def wait_mode(gpu, request):
    before = gpu.lib().dp_get_wait_mode()
    gpu.set_wait_mode(request.param)
    yield request.param
    gpu.set_wait_mode(before)


def _dense_4m():
    desc, data = _mlp_desc(4, 1024, 1)                          # bench.py's Dense-4M: the same model seed
    return desc, data, np.random.Generator(np.random.PCG64(2024)).integers(0, 128, size=(16, 1024)).astype(np.int64)


def _base(gpu, name):
    """(base context, desc, data, inputs); the 2x64 MLP goes through ZkmlContext, the n x Dense MLP that bench.py proves"""
    if name == "dense_4m":
        desc, data, xs = _dense_4m()
    else:
        desc, data, xs = MODELS[name]()
    if name in ("mlp_2x64", "dense_4m"):
        n_layers, width = desc.shape[0] // 3, int(desc[0, 1])
        wb = data.reshape(n_layers, width * width + width)
        ctx = gpu.ZkmlContext(n_layers, width, wb[:, : width * width], wb[:, width * width:], desc[1::3, 1:5])
    else:
        ctx = gpu.ModelContext(desc, data, xs.shape[1])
    return ctx, desc, data, xs


def _check_stacked(gpu, name, rows, n, verify=True):
    """prove n inputs `rows` per proof; pin every proof to the checker's, every output to prove_batch's and infer_batch's"""
    ctx, desc, data, xs = _base(gpu, name)
    xs = xs[:n]
    sctx = ctx.stacked(rows)
    try:
        R = sctx.R
        sdesc, sdata, _, _ = models.stack_rows(desc, data, xs.shape[1], rows)
        assert np.array_equal(sctx.desc, sdesc) and sctx.output_len == R * ctx.output_len
        groups = [xs[g: g + rows] for g in range(0, n, rows)]
        exp = [O.model_prove(sdesc, sdata, models.pad_rows(g, R))[0] for g in groups]
        sec, proofs, gouts, outputs, status, errors, proof_of, row_of = sctx.prove_stacked(xs, N_WORKERS, stride=exp[0].size + 64)
        assert sec > 0 and (status == 0).all() and errors == [None] * n, errors
        assert len(proofs) == len(groups) and gouts.shape == (len(groups), R * ctx.output_len)
        assert proof_of.tolist() == [j // rows for j in range(n)] and row_of.tolist() == [j % rows for j in range(n)]
        for g, p in enumerate(exp):
            assert proofs[g].size == p.size, "%s rows=%d: proof %d has %d words, the checker's %d" % (name, rows, g, proofs[g].size, p.size)
            if not (proofs[g] == p).all():
                raise AssertionError("%s rows=%d: proof %d first differs at word %d of %d" % (name, rows, g, int(np.argmax(proofs[g] != p)), p.size))
            x = models.pad_rows(groups[g], R)
            assert np.array_equal(gouts[g], M.model_output(sdesc, sdata, x))
            if verify:
                assert M.model_verify_output(sdesc, sdata, x, gouts[g]) is None, "%s rows=%d: group %d" % (name, rows, g)
        _, _, want, st, _ = ctx.prove_batch(xs, N_WORKERS)
        assert (st == 0).all() and np.array_equal(outputs, want)
        assert np.array_equal(outputs, ctx.infer_batch(xs)[1])
    finally:
        sctx.free()
        ctx.free()


@pytest.mark.parametrize("wait_mode", [0, 1], indirect=True, ids=["spin", "blocking"])
@pytest.mark.parametrize("name,rows,n", [("mlp_2x64", 4, 7), ("mlp_2x64", 8, 8), ("iris_calibrated", 30, 30), ("token_mlp", 2, 5)])
def test_stacked_equals_checker(gpu, wait_mode, name, rows, n):
    _check_stacked(gpu, name, rows, n, verify=wait_mode == 0)


@pytest.mark.parametrize("wait_mode", [1], indirect=True, ids=["blocking"])
def test_stacked_equals_checker_blake(gpu, wait_mode):
    O.set_hash_mode(1); gpu.set_hasher(1)
    try:
        _check_stacked(gpu, "mlp_2x64", 4, 7)
    finally:
        O.set_hash_mode(0); gpu.set_hasher(0)


@pytest.mark.parametrize("wait_mode", [0], indirect=True, ids=["spin"])
def test_dense_4m_stacked_equals_checker(gpu, wait_mode):
    """Dense-4M at R = 8: one full group and one copy-padded group"""
    _check_stacked(gpu, "dense_4m", 8, 13, verify=False)


@pytest.mark.parametrize("wait_mode", [0, 1], indirect=True, ids=["spin", "blocking"])
def test_screened_input_is_left_out(gpu, wait_mode):
    """the 2x64 MLP with its first requant's input bound cut to 2^14 (as test_gpu_infer_batch does): inputs in [-1, 1] pass it and
    full-range input 2 overflows it; input 5 holds a value of 200, outside the 8-bit domain.  Both are screened out with infer_batch's
    status and message and are not proved; the other inputs are proved in two groups (the second copy-padded), and the stacked handle
    proves a normal batch afterwards"""
    desc, data = _mlp_desc()
    desc = desc.copy()
    desc[1, 4] = 14
    rng = np.random.Generator(np.random.PCG64(21))
    xs = rng.integers(-1, 2, size=(7, 64)).astype(np.int64)
    xs[2] = rng.integers(-127, 128, size=64)
    xs[5, 3] = 200
    ctx = gpu.ModelContext(desc, data, 64)
    sctx = ctx.stacked(4)
    try:
        _, _, st_inf, err_inf = ctx.infer_batch(xs)
        assert [j for j in range(7) if st_inf[j] != 0] == [2, 5]
        assert "requantisation" in err_inf[2] and "outside [-128, 127]" in err_inf[5]
        sdesc, sdata, _, R = models.stack_rows(desc, data, 64, 4)
        groups = [xs[[0, 1, 3, 4]], xs[[6]]]
        exp = [O.model_prove(sdesc, sdata, models.pad_rows(g, R))[0] for g in groups]
        _, proofs, gouts, outputs, status, errors, proof_of, row_of = sctx.prove_stacked(xs, N_WORKERS, stride=exp[0].size + 64)
        assert status.tolist() == st_inf.tolist() and errors == err_inf
        assert proof_of.tolist() == [0, 0, -1, 0, 0, -1, 1] and row_of.tolist() == [0, 1, -1, 2, 3, -1, 0]
        assert not outputs[[2, 5]].any()
        assert len(proofs) == 2 and all((proofs[g] == exp[g]).all() for g in range(2))
        keep = [0, 1, 3, 4, 6]
        assert np.array_equal(outputs[keep], np.stack([M.model_output(desc, data, xs[j]) for j in keep]))
        _, proofs, _, _, status, errors, _, _ = sctx.prove_stacked(xs[keep[:4]], N_WORKERS, stride=exp[0].size + 64)
        assert (status == 0).all() and len(proofs) == 1 and (proofs[0] == exp[0]).all()
    finally:
        sctx.free()
        ctx.free()


def test_prove_stacked_float_iris(gpu):
    """the checker's outputs, and the argmax agreement prove_batch_float gives on the same samples"""
    floats = samples("mlp-iris-01")[0]
    ctx = gpu.ModelContext.from_onnx(os.path.join(GOLDEN, "mlp-iris-01.onnx"), calibration=floats)
    desc, data, xq = iris(True)
    sctx = ctx.stacked(30)
    try:
        assert sctx.metadata is ctx.metadata
        proofs, gouts, outputs, fl, status, errors, proof_of, _ = sctx.prove_stacked_float(floats, N_WORKERS)
        assert (status == 0).all() and len(proofs) == 1 and (proof_of == 0).all()
        assert np.array_equal(outputs, np.stack([M.model_output(desc, data, x) for x in xq]))
        _, b_outputs, b_fl, b_status, _ = ctx.prove_batch_float(floats, N_WORKERS)
        assert (b_status == 0).all() and np.array_equal(outputs, b_outputs) and np.array_equal(fl, b_fl)
        assert fl.shape == (30, ctx.metadata.output_len)
    finally:
        sctx.free()
        ctx.free()


def test_busy_pool_refused(gpu):
    """a second prove_stacked on the stacked handle while its pool is busy is refused as prove_batch refuses it"""
    ctx, _, _, xs = _base(gpu, "mlp_2x64")
    sctx = ctx.stacked(2)
    try:
        sctx.prove_stacked(xs[:2], 1)                              # sizes the default stride, so the thread's call goes to the pool
        res = {}

        def long_call():                                           # screening runs on the calling thread, which needs its own init
            gpu.init(0)
            res.update(r=sctx.prove_stacked(np.repeat(xs, 16, axis=0), 1))
        t = threading.Thread(target=long_call)
        t.start()
        time.sleep(0.5)
        with pytest.raises(gpu.DpError) as e:
            sctx.prove_stacked(xs[:2], 1)
        t.join()
        assert e.value.code == gpu.DP_ERR_STATE and "busy" in str(e.value)
        assert (res["r"][4] == 0).all()
    finally:
        sctx.free()
        ctx.free()


def test_dense_4m_r64_smoke(gpu):
    """Dense-4M at R = 64: the device proves it and the verifier accepts the output matrix it returns"""
    ctx, desc, data, _ = _base(gpu, "dense_4m")
    xs = np.random.Generator(np.random.PCG64(2025)).integers(0, 128, size=(64, 1024)).astype(np.int64)
    sctx = ctx.stacked(64)
    try:
        _, proofs, gouts, outputs, status, errors, _, _ = sctx.prove_stacked(xs, 1, stride=1 << 24)
        assert (status == 0).all(), errors
        sdesc, sdata, _, _ = models.stack_rows(desc, data, 1024, 64)
        assert M.model_verify_output(sdesc, sdata, xs.reshape(-1), gouts[0]) is None
        assert np.array_equal(outputs, ctx.infer_batch(xs)[1])
        print("Dense-4M R=64: one proof of %d words (%.0f words per input)" % (proofs[0].size, proofs[0].size / 64))
    finally:
        sctx.free()
        ctx.free()
