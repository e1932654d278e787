"""StackedContext.open_stream on the H100: arriving inputs grouped into stacked proofs.  Submitted in multiples of `rows`, every stream
proof and public output equals prove_stacked's on the same inputs word for word; a lone group closes on its deadline; a screened-out
input fails alone with infer_batch's message; both handles are held while the stream is open and released when it closes."""
import os
import threading
import time

import numpy as np
import pytest

import models
import oracle_model_io as M
import oracle_py as O
from test_gpu_prove_batch import _mlp_desc
from test_gpu_prove_stacked import _base
from test_stack_rows import GOLDEN, iris, samples

pytestmark = pytest.mark.gpu
N_WORKERS = 4


@pytest.fixture()
def wait_mode(gpu, request):
    before = gpu.lib().dp_get_wait_mode()
    gpu.set_wait_mode(request.param)
    yield request.param
    gpu.set_wait_mode(before)


def _collect(s, n, timeout=600):
    rs = [s.next(timeout) for _ in range(n)]
    return sorted(rs, key=lambda r: r.ticket)


def _stream_equals_stacked(gpu, name, rows, n, verify):
    ctx, desc, data, xs = _base(gpu, name)
    xs = np.concatenate([xs] * (-(-n // len(xs))))[:n] if len(xs) < n else xs[:n]
    sctx = ctx.stacked(rows)
    try:
        _, proofs, gouts, outputs, status, errors, _, _ = sctx.prove_stacked(xs, N_WORKERS)
        assert (status == 0).all(), errors
        want = ctx.infer_batch(xs)[1]
        with sctx.open_stream(N_WORKERS, max_wait=60.0) as s:
            assert s.submit(xs).tolist() == list(range(n))
            rs = _collect(s, n)
        R = sctx.R
        for r in rs:
            assert r.status == 0 and r.error is None, r.error
            assert (r.proof_id, r.row) == (r.ticket // rows, r.ticket % rows)
            p = proofs[r.proof_id]
            assert r.proof.size == p.size and (r.proof == p).all(), "%s rows=%d: proof %d differs from prove_stacked's" % (name, rows, r.proof_id)
            assert r.public_output.shape == (R, ctx.output_len) and np.array_equal(r.public_output.reshape(-1), gouts[r.proof_id])
            assert np.array_equal(r.output, want[r.ticket]) and np.array_equal(r.output, outputs[r.ticket])
        if verify:
            sdesc, sdata, _, _ = models.stack_rows(desc, data, xs.shape[1], rows)
            for g in range(n // rows):
                x = models.pad_rows(xs[g * rows: (g + 1) * rows], R)
                pub = rs[g * rows].public_output.reshape(-1)
                assert M.model_verify_output(sdesc, sdata, x, pub) is None
                bad = pub.copy()
                bad[1] += 1
                assert M.model_verify_output(sdesc, sdata, x, bad) is not None, "the verifier accepted a changed output"
    finally:
        sctx.free()
        ctx.free()


@pytest.mark.parametrize("wait_mode", [0, 1], indirect=True, ids=["spin", "blocking"])
@pytest.mark.parametrize("name,rows,n", [("mlp_2x64", 4, 8), ("mlp_2x64", 8, 16), ("iris_calibrated", 30, 30), ("token_mlp", 2, 4)])
def test_stream_equals_prove_stacked(gpu, wait_mode, name, rows, n):
    _stream_equals_stacked(gpu, name, rows, n, verify=name == "mlp_2x64" and wait_mode == 0)


@pytest.mark.parametrize("wait_mode", [1], indirect=True, ids=["blocking"])
def test_stream_equals_prove_stacked_blake(gpu, wait_mode):
    O.set_hash_mode(1); gpu.set_hasher(1)
    try:
        _stream_equals_stacked(gpu, "mlp_2x64", 4, 8, verify=True)
    finally:
        O.set_hash_mode(0); gpu.set_hasher(0)


@pytest.mark.parametrize("wait_mode", [0], indirect=True, ids=["spin"])
def test_dense_4m_stream_equals_prove_stacked(gpu, wait_mode):
    _stream_equals_stacked(gpu, "dense_4m", 8, 16, verify=False)


def test_deadline_closes_a_short_group(gpu):
    """3 inputs with rows = 8 come back as one proof equal to prove_stacked's on them; a lone input's latency stays under max_wait + 2 x
    one prove_stacked of one input + 20 ms"""
    ctx, _, _, xs = _base(gpu, "mlp_2x64")
    sctx = ctx.stacked(8)
    max_wait = 0.05
    try:
        sctx.prove_stacked(np.repeat(xs, 12, axis=0), N_WORKERS)      # 12 groups: every worker thread has proved once
        _, proofs3, _, _, st, _, _, _ = sctx.prove_stacked(xs[:3], N_WORKERS)
        assert (st == 0).all()
        one = []
        for _ in range(3):
            t0 = time.perf_counter()
            _, proofs1, _, _, st, _, _, _ = sctx.prove_stacked(xs[3:4], N_WORKERS)
            one.append(time.perf_counter() - t0)
        with sctx.open_stream(N_WORKERS, max_wait=max_wait) as s:
            s.submit(xs[:3])
            rs = _collect(s, 3)
            assert [(r.proof_id, r.row) for r in rs] == [(0, 0), (0, 1), (0, 2)] and all(r.status == 0 for r in rs)
            assert (rs[0].proof == proofs3[0]).all()
            lone = []
            for _ in range(3):
                t0 = time.perf_counter()
                s.submit(xs[3])
                r = s.next(60)
                lone.append(time.perf_counter() - t0)
                assert r.status == 0 and r.row == 0 and (r.proof == proofs1[0]).all()
        print("prove_stacked of one input %.1f ms, lone stream input %s ms" % (1e3 * np.median(one), ["%.1f" % (1e3 * v) for v in lone]))
        assert max(lone) < max_wait + 2 * np.median(one) + 0.02, (lone, one)
        assert min(lone) >= max_wait, lone
    finally:
        sctx.free()
        ctx.free()


@pytest.mark.parametrize("wait_mode", [0, 1], indirect=True, ids=["spin", "blocking"])
def test_screened_input_fails_alone(gpu, wait_mode):
    """the 2x64 MLP with its first requant's input bound cut to 2^14: input 2 overflows it and input 5 holds 200.  Both fail with
    infer_batch's status and message; groups [0, 1, 3] and [4, 6, 7] are proved as the checker proves them (not topped up).  The
    stacked context has measured no proof yet, so the stream sizes its stride on the first group."""
    desc, data = _mlp_desc()
    desc = desc.copy()
    desc[1, 4] = 14
    rng = np.random.Generator(np.random.PCG64(21))
    xs = rng.integers(-1, 2, size=(8, 64)).astype(np.int64)
    xs[2] = rng.integers(-127, 128, size=64)
    xs[5, 3] = 200
    ctx = gpu.ModelContext(desc, data, 64)
    sctx = ctx.stacked(4)
    try:
        _, want, st_inf, err_inf = ctx.infer_batch(xs)
        with sctx.open_stream(N_WORKERS, max_wait=60.0) as s:
            s.submit(xs)
            rs = _collect(s, 8)
        assert [r.status for r in rs] == st_inf.tolist() and [r.error for r in rs] == err_inf
        assert [(r.proof_id, r.row) for r in rs] == [(0, 0), (0, 1), (-1, -1), (0, 2), (1, 0), (-1, -1), (1, 1), (1, 2)]
        sdesc, sdata, _, R = models.stack_rows(desc, data, 64, 4)
        for g, idx in enumerate([[0, 1, 3], [4, 6, 7]]):
            exp = O.model_prove(sdesc, sdata, models.pad_rows(xs[idx], R))[0]
            assert (rs[idx[0]].proof == exp).all()
            for j in idx:
                assert np.array_equal(rs[j].output, want[j])
        assert rs[2].proof.size == 0 and not rs[5].output.any()
    finally:
        sctx.free()
        ctx.free()


def test_float_inputs_iris(gpu):
    floats = samples("mlp-iris-01")[0]
    ctx = gpu.ModelContext.from_onnx(os.path.join(GOLDEN, "mlp-iris-01.onnx"), calibration=floats)
    sctx = ctx.stacked(30)
    try:
        proofs, gouts, outputs, fl, status, _, _, _ = sctx.prove_stacked_float(floats, N_WORKERS)
        assert (status == 0).all()
        with sctx.open_stream(N_WORKERS, max_wait=60.0) as s:
            s.submit_float(floats)
            rs = _collect(s, 30)
        assert all(r.status == 0 and r.proof_id == 0 for r in rs) and (rs[0].proof == proofs[0]).all()
        assert np.array_equal(np.stack([r.output for r in rs]), outputs) and np.array_equal(np.stack([r.output_float for r in rs]), fl)
        assert np.array_equal(outputs, np.stack([M.model_output(*iris(True)[:2], x) for x in iris(True)[2]]))
    finally:
        sctx.free()
        ctx.free()


def test_handles_are_held_and_released(gpu):
    ctx, _, _, xs = _base(gpu, "mlp_2x64")
    sctx, other = ctx.stacked(4), ctx.stacked(2)
    try:
        with pytest.raises(ValueError):
            sctx.open_stream(0, 0.02)
        with pytest.raises(ValueError):
            sctx.open_stream(2, -1.0)
        with pytest.raises(ValueError):
            sctx.open_stream(2, 0.02, capacity=3)
        p = ctx.open_stream(2, capacity=8)                       # a ProofStream on the base: its pool is busy
        with pytest.raises(gpu.DpError) as e:
            sctx.open_stream(2, 0.02)
        assert e.value.code == gpu.DP_ERR_STATE
        p.close()
        s = sctx.open_stream(N_WORKERS, 0.02)
        calls = [lambda: ctx.prove_batch(xs[:2], 2), lambda: ctx.infer_batch(xs[:2]), lambda: ctx.open_stream(2),
                 lambda: ctx.prove_concurrent(2, 2), lambda: sctx.prove_batch(np.tile(xs[:1], (1, 4)), 2),
                 lambda: sctx.prove_stacked(xs[:2], 2), lambda: sctx.open_stream(2, 0.02), lambda: other.prove_stacked(xs[:2], 2),
                 lambda: other.open_stream(2, 0.02)]
        for call in calls:
            with pytest.raises(gpu.DpError) as e:
                call()
            assert e.value.code == gpu.DP_ERR_STATE and "busy" in str(e.value)
        s.submit(xs[:4])
        assert all(r.status == 0 for r in _collect(s, 4))
        assert s.close() == 0
        assert (ctx.infer_batch(xs)[2] == 0).all()
        assert (other.prove_stacked(xs[:2], 2)[4] == 0).all()
        # freeing the base with a stream open closes it first
        s = sctx.open_stream(N_WORKERS, 0.02)
        s.submit(xs[:8])
        t = threading.Thread(target=ctx.free)
        t.start()
        t.join(120)
        assert not t.is_alive(), "freeing the base with an open stacked stream did not return"
        with pytest.raises(gpu.DpError):
            s.next(0)
    finally:
        other.free()
        sctx.free()
        ctx.free()


def test_close_while_proofs_run(gpu):
    ctx, _, _, xs = _base(gpu, "mlp_2x64")
    sctx = ctx.stacked(4)
    try:
        s = sctx.open_stream(N_WORKERS, max_wait=0.01, capacity=512)
        s.submit(np.repeat(xs, 50, axis=0))                      # 400 inputs, 100 groups
        r = s.next(120)
        assert r.status == 0
        cancelled = s.close()
        assert 0 < cancelled <= 399, cancelled
        assert s.close() == 0
        _, _, _, _, status, _, _, _ = sctx.prove_stacked(xs[:4], N_WORKERS)
        assert (status == 0).all()
    finally:
        sctx.free()
        ctx.free()


def test_cnn_is_refused_by_stacked(gpu):
    desc, data, x, _ = models.cnn_small(seed=3)
    ctx = gpu.ModelContext(desc, data, x.size)
    try:
        with pytest.raises(ValueError):
            ctx.stacked(4)
    finally:
        ctx.free()
