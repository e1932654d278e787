"""StackedStream's grouping and result bookkeeping, on the CPU: a fake screener (infer_batch's return shape; an input whose first value
is outside [-128, 127] fails) and a fake ProofStream whose "proof" of a group is its ticket and whose output matrix is its input matrix,
so that every result shows which rows went into which proof.  Also the reservation of the base and stacked handles, on contexts made
without a device: every refused call is refused before it reaches the library."""
import threading
import time

import numpy as np
import pytest

import dpb200 as dp
import models

L = 4           # input (and, for the fake prover, output) length


class Screener:
    def __init__(self):
        self.calls = []

    def __call__(self, x):
        self.calls.append(x.copy())
        bad = np.abs(x[:, 0]) > 127
        return 1e-4, x.copy(), np.where(bad, dp.DP_ERR_INVALID, 0).astype(np.int32), ["value out of range" if b else None for b in bad]


class Prover:
    """ProofStream-like: jobs finish in submission order, at once unless `hold` keeps them queued; tickets in `fail` fail"""

    def __init__(self, hold=False, fail=()):
        self.cv, self.hold, self.fail = threading.Condition(), hold, set(fail)
        self.jobs, self.queued, self.done, self.closed = [], [], [], False

    def submit(self, x):
        with self.cv:
            self.jobs.append(np.array(x))
            self.queued.append(len(self.jobs) - 1)
            self.cv.notify_all()
            return np.array([len(self.jobs) - 1], dtype=np.uint64)

    def release(self):
        with self.cv:
            self.hold = False
            self.cv.notify_all()

    def next(self, timeout=None):
        end = None if timeout is None else time.monotonic() + timeout
        with self.cv:
            while True:
                if self.closed:
                    raise dp.DpError(dp.DP_ERR_STATE, "closed")
                if not self.hold:
                    self.done += self.queued
                    self.queued = []
                if self.done:
                    t = self.done.pop(0)
                    if t in self.fail:
                        return dp.StreamResult(t, np.zeros(0, np.uint64), np.zeros_like(self.jobs[t]), dp.DP_ERR_INVALID, "proof failed", None)
                    return dp.StreamResult(t, np.full(3, t, dtype=np.uint64), self.jobs[t].copy(), 0, None, None)
                if not self.queued:
                    raise dp.DpError(dp.DP_ERR_STATE, "nothing to collect")
                left = None if end is None else end - time.monotonic()
                if left is not None and left <= 0:
                    raise dp.StreamTimeout(dp.DP_ERR_TIMEOUT, "timeout")
                self.cv.wait(left)

    def close(self):
        with self.cv:
            self.closed, n, self.queued = True, len(self.queued), []
            self.cv.notify_all()
            return n


def stream(rows=4, R=4, max_wait=60.0, capacity=None, prover=None, metadata=None):
    """(stream, screener, prover, list of the inputs open_prover was called with)"""
    scr, pr, opened = Screener(), prover or Prover(), []

    def open_prover(x):
        opened.append(x)
        return pr
    s = dp.StackedStream(rows, R, L, L, 2, max_wait, capacity, scr, open_prover, metadata)
    return s, scr, pr, opened


def inputs(n, seed=0):
    return np.random.Generator(np.random.PCG64(seed)).integers(-128, 128, size=(n, L)).astype(np.int64)


def collect(s, n, timeout=5.0):
    return [s.next(timeout) for _ in range(n)]


def wait_until(cond, timeout=5.0):
    end = time.monotonic() + timeout
    while not cond():
        assert time.monotonic() < end, "condition not reached"
        time.sleep(0.005)


def test_group_closes_at_rows_in_ticket_order():
    s, scr, pr, opened = stream()
    with s:
        xs = inputs(8)
        assert s.submit(xs[:3]).tolist() == [0, 1, 2]
        assert s.submit(xs[3:]).tolist() == [3, 4, 5, 6, 7]
        got = sorted(collect(s, 8), key=lambda r: r.ticket)
        assert [r.ticket for r in got] == list(range(8))
        assert [r.proof_id for r in got] == [0] * 4 + [1] * 4 and [r.row for r in got] == [0, 1, 2, 3] * 2
        assert len(pr.jobs) == 2 and len(opened) == 1 and np.array_equal(opened[0], pr.jobs[0])
        for g in range(2):
            assert np.array_equal(pr.jobs[g], xs[4 * g: 4 * g + 4].reshape(-1))
            assert np.array_equal(scr.calls[g], xs[4 * g: 4 * g + 4])              # one screening call per group
        for r in got:
            assert r.status == 0 and r.error is None and r.output_float is None
            assert np.array_equal(r.output, xs[r.ticket]) and r.public_output.shape == (4, L)
            assert r.proof.tolist() == [r.proof_id] * 3
        assert got[0].proof is got[3].proof and got[0].public_output is got[1].public_output   # shared by the group
        with pytest.raises(dp.DpError) as e:
            s.next(5.0)
        assert e.value.code == dp.DP_ERR_STATE


def test_group_closes_after_max_wait_and_not_before():
    s, _, pr, _ = stream(rows=8, R=8, max_wait=0.4)
    with s:
        xs = inputs(3)
        t0 = time.monotonic()
        s.submit(xs)
        time.sleep(0.2)
        assert pr.jobs == []                                   # 0.2 s after the submit: still waiting for company
        rs = collect(s, 3)
        waited = time.monotonic() - t0
        assert 0.4 <= waited < 3.0, waited
        assert len(pr.jobs) == 1 and sorted(r.row for r in rs) == [0, 1, 2] and {r.proof_id for r in rs} == {0}
        # padding rows copy the last input of the group
        assert np.array_equal(pr.jobs[0], models.pad_rows(xs, 8))
        assert np.array_equal(rs[0].public_output[3:], np.repeat(xs[2:], 5, axis=0))


def test_groups_are_not_topped_up():
    """a screened-out input leaves a hole that later arrivals do not fill; a group closed on its deadline is not joined by inputs
    submitted after it closed"""
    s, _, pr, _ = stream(max_wait=0.1)
    with s:
        xs = inputs(8)
        xs[1, 0] = 500
        s.submit(xs)
        rs = {r.ticket: r for r in collect(s, 8)}
        assert np.array_equal(pr.jobs[0], models.pad_rows(xs[[0, 2, 3]], 4)) and np.array_equal(pr.jobs[1], xs[4:].reshape(-1))
        assert [rs[j].row for j in range(8)] == [0, -1, 1, 2, 0, 1, 2, 3]
        s.submit(xs[:2][[0]])
        wait_until(lambda: len(pr.jobs) == 3)
        s.submit(xs[[2, 3]])
        collect(s, 3)
        assert np.array_equal(pr.jobs[2], models.pad_rows(xs[:1], 4)) and np.array_equal(pr.jobs[3], models.pad_rows(xs[[2, 3]], 4))


def test_screened_out_input_comes_back_before_its_groups_proof():
    s, _, pr, _ = stream(prover=Prover(hold=True))
    with s:
        xs = inputs(4)
        xs[2, 0] = -129
        s.submit(xs)
        r = s.next(5.0)
        assert (r.ticket, r.proof_id, r.row, r.status, r.error) == (2, -1, -1, dp.DP_ERR_INVALID, "value out of range")
        assert r.proof.size == 0 and r.public_output.shape == (0, L) and not r.output.any()
        with pytest.raises(dp.StreamTimeout):
            s.next(0.2)                                        # the group's proof is held
        pr.release()
        rs = sorted(collect(s, 3), key=lambda r: r.ticket)
        assert [(r.ticket, r.proof_id, r.row) for r in rs] == [(0, 0, 0), (1, 0, 1), (3, 0, 2)]
        assert np.array_equal(pr.jobs[0], models.pad_rows(xs[[0, 1, 3]], 4))


def test_group_failing_in_the_prover_fails_every_member():
    s, _, _, _ = stream(prover=Prover(fail={0}))
    with s:
        xs = inputs(8)
        s.submit(xs)
        rs = sorted(collect(s, 8), key=lambda r: r.ticket)
        for r in rs[:4]:
            assert (r.status, r.error, r.proof_id, r.proof.size) == (dp.DP_ERR_INVALID, "proof failed", 0, 0) and not r.output.any()
        assert all(r.status == 0 and r.proof_id == 1 for r in rs[4:])


def test_prover_failing_as_a_whole_fails_its_groups():
    """a prover whose next raises (not a job's failure) fails every group still out, so that no caller waits for ever"""
    class Broken(Prover):
        def next(self, timeout=None):
            raise ValueError("prover broke")
    s, _, _, _ = stream(prover=Broken())
    with s:
        s.submit(inputs(4))
        rs = collect(s, 4)
        assert all((r.status, r.error, r.proof_id) == (dp.DP_ERR_INVALID, "prover broke", -1) for r in rs)


def test_all_screened_out_group_submits_nothing():
    s, scr, pr, opened = stream()
    with s:
        xs = inputs(4)
        xs[:, 0] = 300
        s.submit(xs)
        rs = collect(s, 4)
        assert all(r.status == dp.DP_ERR_INVALID and r.proof_id == -1 for r in rs)
        assert len(scr.calls) == 1 and pr.jobs == [] and opened == []
        s.submit(inputs(4, 1))                                  # the next group is proof 0
        assert {r.proof_id for r in collect(s, 4)} == {0}


def test_submit_is_all_or_nothing_against_capacity():
    s, _, pr, _ = stream(rows=2, R=2, capacity=4, prover=Prover(hold=True))
    with s:
        xs = inputs(8)
        assert s.submit(xs[:3]).tolist() == [0, 1, 2]
        t0 = time.monotonic()
        with pytest.raises(dp.StreamTimeout):
            s.submit(xs[3:5], timeout=0.2)
        assert time.monotonic() - t0 >= 0.19
        with pytest.raises(dp.StreamTimeout):
            s.submit(xs[3:5], timeout=0)
        with pytest.raises(dp.DpError) as e:
            s.submit(inputs(5))
        assert e.value.code == dp.DP_ERR_INVALID
        assert s.submit(xs[3], timeout=0).tolist() == [3]       # nothing of the refused submits was taken
        done = []
        t = threading.Thread(target=lambda: done.append(s.submit(xs[4:6], timeout=5.0)))
        t.start()
        time.sleep(0.1)
        assert not done                                         # waits for room
        pr.release()
        first = collect(s, 2)
        t.join(5.0)
        assert done[0].tolist() == [4, 5]
        assert sorted(r.ticket for r in first + collect(s, 4)) == list(range(6))


def test_empty_stream_refuses_next_at_once():
    s, _, _, _ = stream()
    with s:
        t0 = time.monotonic()
        with pytest.raises(dp.DpError) as e:
            s.next()
        assert e.value.code == dp.DP_ERR_STATE and time.monotonic() - t0 < 1.0
        assert list(s.results()) == []


def test_concurrent_callers_get_every_result_once():
    s, _, _, _ = stream(rows=4, R=4, max_wait=0.05, capacity=256)
    with s:
        xs = inputs(200)
        subs = [threading.Thread(target=lambda k=k: [s.submit(xs[k + 4 * j], timeout=10) for j in range(50)]) for k in range(4)]
        for t in subs:
            t.start()
        for t in subs:
            t.join()
        got, lock = [], threading.Lock()

        def take():
            for r in s.results(timeout=10):
                with lock:
                    got.append(r)
        ts = [threading.Thread(target=take) for _ in range(4)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert sorted(r.ticket for r in got) == list(range(200))
        for r in got:
            assert r.status == 0 and r.public_output[r.row] is not None


def test_close_cancels_pending_inputs_and_groups():
    s, _, pr, _ = stream(prover=Prover(hold=True))
    xs = inputs(11)
    s.submit(xs[:8])
    wait_until(lambda: len(pr.jobs) == 2)                      # two groups queued in the prover, held
    s.submit(xs[8:])                                            # three inputs waiting for company
    assert s.close() == 11
    assert s.close() == 0
    for call in (lambda: s.submit(xs[0]), lambda: s.next(0)):
        with pytest.raises(dp.DpError) as e:
            call()
        assert e.value.code == dp.DP_ERR_STATE
    s, _, pr, _ = stream()
    s.submit(xs[:4])
    wait_until(lambda: len(pr.done) == 0 and len(pr.jobs) == 1 and not pr.queued)
    s.submit(xs[4:7])
    assert s.close() == 3                                       # the finished group's results are dropped, not cancelled


def test_float_inputs_use_the_metadata():
    class Md:
        def quantize_input(self, f):
            return np.rint(np.asarray(f) * 100).astype(np.int64)

        def dequantize_output(self, y):
            return np.asarray(y, dtype=np.float32) / 100
    s, _, _, _ = stream(metadata=Md())
    with s:
        f = np.full((4, L), 0.5, dtype=np.float32)
        s.submit_float(f)
        for r in collect(s, 4):
            assert r.output.tolist() == [50] * L and np.allclose(r.output_float, 0.5)
    s, _, _, _ = stream()
    with s, pytest.raises(ValueError):
        s.submit_float(np.zeros((1, L), dtype=np.float32))


@pytest.mark.parametrize("kw", [dict(n_workers=0), dict(max_wait=-0.001), dict(max_wait=float("nan")), dict(max_wait=float("inf")),
                                dict(capacity=3)])
def test_open_refusals(kw):
    args = dict(n_workers=2, max_wait=0.02, capacity=None)
    args.update(kw)
    opened = []
    with pytest.raises(ValueError):
        dp.StackedStream(4, 4, L, L, args["n_workers"], args["max_wait"], args["capacity"], Screener(), opened.append)
    assert opened == []


def test_submit_refuses_wrong_shapes():
    s, _, _, _ = stream()
    with s:
        for bad in (np.zeros((1, L + 1)), np.zeros((0, L)), np.zeros((1, 1, L)), np.zeros(L - 1)):
            with pytest.raises(ValueError):
                s.submit(bad)
        assert s.submit(np.zeros(L, dtype=np.int64)).tolist() == [0]    # the refused submits took no ticket


def _fake_context():
    """a ZkmlContext without a handle: every call it would pass to the library is refused first, or fails"""
    c = object.__new__(dp.ModelContext)
    c.h, c._mu, c.input_len, c._out = None, threading.Lock(), L, np.zeros(8, dtype=np.uint64)
    return c


def test_handles_are_held_while_open():
    base, sctx, other = _fake_context(), _fake_context(), _fake_context()
    s, _, _, _ = stream()
    s._hold((base, sctx))
    x = np.zeros((1, L), dtype=np.int64)
    for c in (base, sctx):
        for call in (lambda: c.infer_batch(x), lambda: c.prove_batch(x, 1), lambda: c.open_stream(1), lambda: c.prove_concurrent(1, 1),
                     lambda: c.prove_concurrent_all(1, 1, 8)):
            with pytest.raises(dp.DpError) as e:
                call()
            assert e.value.code == dp.DP_ERR_STATE and "busy" in str(e.value)
    t, _, _, _ = stream()
    for pair in ((base, other), (other, sctx)):                  # a second stream on either handle
        with pytest.raises(dp.DpError) as e:
            t._hold(pair)
        assert e.value.code == dp.DP_ERR_STATE
    assert other._holder is None
    s.close()
    assert base._holder is None and sctx._holder is None
    t._hold((base, sctx))
    t.close()
    # a busy pool: a call in progress, or an open ProofStream
    base._calls = 1
    with pytest.raises(dp.DpError):
        t._hold((base, sctx))
    base._calls, sctx._stream = 0, object()
    with pytest.raises(dp.DpError):
        t._hold((base, sctx))
    assert base._holder is None and sctx._holder is None
