"""Proof streams (ZkmlContext.open_stream, dph_zkml_stream_*) on the H100: every stream proof and output equals prove_batch's for the
same input and label, word for word, under both hashers; the 2x64 MLP's also equal the checker's and the restated verifier accepts
them.  A failing input fails alone, a too-small stride fails only the jobs whose proof is longer, concurrent submitters and a
collector see every ticket once, the pool is held and released, and a lone job on an idle stream is not delayed."""
import os
import threading
import time

import numpy as np
import pytest

import oracle_model_io as M
import oracle_py as O
from test_gpu_prove_batch import _model
from test_onnx_calibration import GOLDEN, samples

pytestmark = pytest.mark.gpu
N_WORKERS = 4
SPLITS = (1, 3, 2)          # submit sizes: the six inputs in three calls


def _collect(stream):
    """{ticket: StreamResult} of everything submitted so far"""
    got = {}
    for r in stream.results():
        assert r.ticket not in got, "ticket %d delivered twice" % r.ticket
        got[r.ticket] = r
    return got


def _submit_in_parts(stream, xs, submit):
    tickets, k = [], 0
    for n in SPLITS:
        tickets += list(submit(xs[k:k + n]))
        k += n
    assert k == len(xs) and tickets == list(range(tickets[0], tickets[0] + len(xs)))
    return tickets


def _context(gpu, name):
    """(ctx, xs, desc, data): xs quantised inputs, or float samples for the calibrated CIFAR model"""
    if name == "cnn-cifar-01":
        xs = samples(name)[0]
        return gpu.ModelContext.from_onnx(os.path.join(GOLDEN, name + ".onnx"), calibration=xs), xs[:6], None, None
    desc, data, xs = _model(name)
    return gpu.ModelContext(desc, data, xs.shape[1]), xs, desc, data


@pytest.mark.parametrize("hasher", [0, 1], ids=["poseidon2", "blake3"])
@pytest.mark.parametrize("name", ["mlp_2x64", "cnn_small", "cnn-cifar-01"])
def test_stream_equals_prove_batch(gpu, name, hasher):
    O.set_hash_mode(hasher); gpu.set_hasher(hasher)
    ctx, xs, desc, data = _context(gpu, name)
    try:
        is_float = name == "cnn-cifar-01"
        if is_float:
            proofs, outputs, floats, status, _ = ctx.prove_batch_float(xs, N_WORKERS, label=b"stream-test")
        else:
            _, proofs, outputs, status, _ = ctx.prove_batch(xs, N_WORKERS, label=b"stream-test")
        assert (status == 0).all()
        with ctx.open_stream(N_WORKERS, label=b"stream-test") as s:
            tickets = _submit_in_parts(s, xs, s.submit_float if is_float else s.submit)
            got = _collect(s)
        assert sorted(got) == tickets
        for j, t in enumerate(tickets):
            r = got[t]
            assert r.status == 0 and r.error is None
            assert r.proof.size == proofs[j].size and np.array_equal(r.proof, proofs[j]), "%s: stream proof of input %d differs" % (name, j)
            assert np.array_equal(r.output, outputs[j]), "%s: stream output of input %d differs" % (name, j)
            if is_float:
                assert np.array_equal(r.output_float, floats[j])
            else:
                assert r.output_float is None
        if name == "mlp_2x64":             # and the checker: its proofs, its inference, and the restated verifier on the device output
            for j, t in enumerate(tickets):
                assert np.array_equal(got[t].proof, O.model_prove(desc, data, xs[j], label=b"stream-test")[0])
                assert np.array_equal(got[t].output, M.model_output(desc, data, xs[j]))
                assert M.model_verify_output(desc, data, xs[j], got[t].output, label=b"stream-test") is None
    finally:
        ctx.free()
        O.set_hash_mode(0); gpu.set_hasher(0)


def test_failing_input_and_short_stride_fail_alone(gpu):
    """input 2, scaled out of the quantised range, fails with prove_batch's status and message; with a stride one word short of a
    proof every proved job fails alone with DP_ERR_INVALID, the failing input keeps its own message, and the stream goes on"""
    ctx, xs, _, _ = _context(gpu, "mlp_2x64")
    try:
        bad = xs.copy()
        bad[2] *= 4096
        _, proofs, outputs, status, errors = ctx.prove_batch(bad, N_WORKERS)
        assert [j for j in range(len(xs)) if status[j]] == [2]
        words = proofs[0].size
        with ctx.open_stream(N_WORKERS, stride=words) as s:
            got = _collect_after(s, s.submit(bad))
            for j in range(len(xs)):
                assert got[j].status == status[j] and got[j].error == errors[j]
                assert np.array_equal(got[j].proof, proofs[j]) and np.array_equal(got[j].output, outputs[j])
        with ctx.open_stream(N_WORKERS, stride=words - 1) as s:
            got = _collect_after(s, s.submit(bad))
            assert got[2].status == status[2] and got[2].error == errors[2]
            for j in (0, 1, 3, 4, 5):
                assert got[j].status == gpu.DP_ERR_INVALID and "longer than the stream's stride" in got[j].error
                assert got[j].proof.size == 0 and not got[j].output.any()
            got = _collect_after(s, s.submit(xs[:1]))
            assert got[6].status == gpu.DP_ERR_INVALID, "the stream serves jobs after the failures"
    finally:
        ctx.free()


def _collect_after(stream, tickets):
    got = _collect(stream)
    assert sorted(got) == [int(t) for t in tickets]
    return got


def test_two_submitters_and_a_collector(gpu):
    ctx, xs, _, _ = _context(gpu, "mlp_2x64")
    try:
        _, proofs, _, _, _ = ctx.prove_batch(xs, N_WORKERS)
        per = 12
        with ctx.open_stream(N_WORKERS, capacity=8) as s:
            sent, lock, got = {}, threading.Lock(), []

            def produce(seed):
                rng = np.random.Generator(np.random.PCG64(seed))
                k = 0
                while k < per:
                    idx = rng.integers(0, len(xs), size=int(min(rng.integers(1, 4), per - k)))
                    t = s.submit(xs[idx])
                    with lock:
                        sent.update(zip(t.tolist(), idx.tolist()))
                    k += idx.size

            def collect():
                while len(got) < 2 * per:
                    try:
                        got.append(s.next(timeout=0.05))
                    except gpu.StreamTimeout:
                        pass
                    except gpu.DpError as e:
                        assert e.code == gpu.DP_ERR_STATE       # momentarily nothing submitted
                        time.sleep(0.01)
            th = [threading.Thread(target=produce, args=(k,)) for k in (1, 2)] + [threading.Thread(target=collect)]
            for t in th:
                t.start()
            for t in th:
                t.join(120)
            assert not any(t.is_alive() for t in th)
        assert sorted(r.ticket for r in got) == list(range(2 * per))
        for r in got:
            assert r.status == 0 and np.array_equal(r.proof, proofs[sent[r.ticket]])
    finally:
        ctx.free()


def test_pool_is_held_and_released(gpu):
    """open refusals on a real handle; prove_batch, infer_batch and a second open are refused while a stream is open and work after
    close; close with a backlog cancels jobs and leaves the handle usable; freeing a context with an open stream returns"""
    import ctypes as C
    ctx, xs, _, _ = _context(gpu, "cnn_small")
    H = gpu.host()
    try:
        h = C.c_void_p()
        assert H.dph_zkml_stream_open(None, 0, 2, b"m2vec", 64, 4, C.byref(h)) == gpu.DP_ERR_INVALID
        assert H.dph_zkml_stream_open(ctx.h, gpu.device_count(), 2, b"m2vec", 64, 4, C.byref(h)) == gpu.DP_ERR_INVALID
        assert b"out of range" in H.dph_last_error()
        s = ctx.open_stream(2, capacity=64)
        for call in (lambda: ctx.prove_batch(xs, 2), lambda: ctx.infer_batch(xs), lambda: ctx.open_stream(2)):
            with pytest.raises(gpu.DpError) as e:
                call()
            assert e.value.code == gpu.DP_ERR_STATE and "busy" in str(e.value)
        with pytest.raises(gpu.DpError) as e:
            s.submit(np.repeat(xs, 11, axis=0))          # 66 > capacity
        assert e.value.code == gpu.DP_ERR_INVALID
        s.submit(np.repeat(xs, 10, axis=0))
        cancelled = s.close()
        assert 0 < cancelled <= 60
        assert s.close() == 0
        _, _, _, status, _ = ctx.prove_batch(xs, 2)
        assert (status == 0).all()
        assert (ctx.infer_batch(xs)[2] == 0).all()
        s = ctx.open_stream(2, capacity=64)
        s.submit(np.repeat(xs, 10, axis=0))
        t = threading.Thread(target=ctx.free)
        t.start()
        t.join(120)
        assert not t.is_alive(), "freeing a context with an open stream did not return"
        assert not s.h
        with pytest.raises(gpu.DpError):
            s.next()
    finally:
        ctx.free()


def test_lone_job_is_not_staggered(gpu):
    """after a large batch has timed the pool (so the stagger rule is armed), a lone job on an idle stream finishes within a small
    factor of one prove(x) on the calling thread"""
    ctx, xs, _, _ = _context(gpu, "cnn_small")
    workers = 16
    try:
        ctx.prove_batch(np.repeat(xs, 8, axis=0), workers)       # 48 jobs, 3 per worker: the stagger rule applies, the pool is timed
        one = []
        for _ in range(3):
            t0 = time.perf_counter(); ctx.prove(xs[0]); one.append(time.perf_counter() - t0)
        with ctx.open_stream(workers) as s:
            lone = []
            for k in range(3):
                t0 = time.perf_counter()
                s.submit(xs[k])
                r = s.next()
                lone.append(time.perf_counter() - t0)
                assert r.status == 0
        print("prove(x) %.1f ms, lone stream job %s ms" % (1e3 * np.median(one), ["%.1f" % (1e3 * v) for v in lone]))
        assert max(lone) < 2.0 * np.median(one) + 0.02
    finally:
        ctx.free()
