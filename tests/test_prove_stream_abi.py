"""CPU tests of the proof stream (dph_zkml_stream_*): the C entry points' refusals, and the stream's queue (host/proof_queue.hpp)
served by host threads that run a fake job (tests/stream_queue_io.cpp): tickets, all-or-nothing submits at capacity, timed waits,
the empty-stream refusal, cancellation at close, and each result delivered exactly once to concurrent callers."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

import dpb200

OK, INVALID, STATE, TIMEOUT = dpb200.DP_OK, dpb200.DP_ERR_INVALID, dpb200.DP_ERR_STATE, dpb200.DP_ERR_TIMEOUT
VP, U64, I64, U32 = C.c_void_p, C.c_uint64, C.c_int64, C.c_uint32
IN_LEN = 3          # the fake job's input: [value (< 0 fails), milliseconds to sleep, anything]


def _p(a):
    return None if a is None else a.ctypes.data_as(VP)


# ---- the C entry points' refusals ---------------------------------------------------------------------------------------------
def _open(handle=None, label=b"m2vec", stream=True, n_workers=2, capacity=4, device=0):
    s = VP()
    return dpb200.host().dph_zkml_stream_open(handle, device, n_workers, label, 64, capacity, C.byref(s) if stream else None)


@pytest.mark.parametrize("case", ["label", "stream", "n_workers", "capacity"])
def test_open_refuses_bad_arguments(case):
    """null arguments, no workers and no capacity are refused before the device is looked at"""
    kw = {"label": dict(label=None), "stream": dict(stream=False), "n_workers": dict(n_workers=0), "capacity": dict(capacity=0)}[case]
    assert _open(**kw) == INVALID
    msg = dpb200.host().dph_last_error().decode()
    assert "dph_zkml_stream_open" in msg and ("null argument" in msg if case in ("label", "stream") else "no workers or no capacity" in msg)


def test_open_without_a_device():
    if dpb200.device_count() > 0:
        pytest.skip("a device is visible: the GPU tests cover the open refusals on a real handle")
    assert _open() == dpb200.DP_ERR_NO_DEVICE
    assert b"no CPU fallback" in dpb200.host().dph_last_error()


def test_submit_next_close_refuse_a_null_stream():
    H = dpb200.host()
    x, first = np.zeros(IN_LEN, dtype=np.int64), U64()
    assert H.dph_zkml_stream_submit(None, _p(x), 1, 0, C.byref(first)) == INVALID
    assert b"dph_zkml_stream_submit: null stream" in H.dph_last_error()
    ticket, plen, st = U64(), U64(), C.c_int32()
    proof, out = np.zeros(8, dtype=np.uint64), np.zeros(8, dtype=np.int64)
    assert H.dph_zkml_stream_next(None, 0, C.byref(ticket), _p(proof), C.byref(plen), _p(out), C.byref(st), None, 0) == INVALID
    assert b"dph_zkml_stream_next: null argument" in H.dph_last_error()
    assert H.dph_zkml_stream_close(None, None) == INVALID
    assert b"dph_zkml_stream_close: null stream" in H.dph_last_error()


# ---- the queue under a fake job ----------------------------------------------------------------------------------------------
_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libdp_stream_queue_io.so")
_q = None


def Q():
    global _q
    if _q is None:
        if not os.path.exists(_PATH):
            raise ImportError("stream queue test library not built: run `make oracle`")
        _q = C.CDLL(_PATH)
        for name, res, args in [("dpq_last_error", C.c_char_p, []), ("dpq_open", VP, [U64, U64, U32]), ("dpq_started", U64, [VP]),
                                ("dpq_submit", C.c_int, [VP, VP, U64, I64, VP]),
                                ("dpq_next", C.c_int, [VP, I64, VP, VP, VP, VP, VP, VP, U64]), ("dpq_close", None, [VP, VP])]:
            f = getattr(_q, name)
            f.restype, f.argtypes = res, args
    return _q


class Fake:
    def __init__(self, capacity, servers):
        self.h = Q().dpq_open(IN_LEN, capacity, servers)

    def submit(self, values, ms=0, timeout=0):
        """one job per value: its input is [value, ms, 0]; -> (rc, first ticket)"""
        x = np.array([[v, ms, 0] for v in values], dtype=np.int64).reshape(-1, IN_LEN)
        first = U64()
        rc = Q().dpq_submit(self.h, _p(x) if len(values) else _p(np.zeros(IN_LEN, dtype=np.int64)), len(values), timeout, C.byref(first))
        return rc, first.value

    def next(self, timeout=-1):
        """-> (rc, (ticket, proof, output, status, message) | None)"""
        ticket, plen, st = U64(), U64(), C.c_int32()
        proof, out = np.zeros(2, dtype=np.uint64), np.zeros(IN_LEN, dtype=np.int64)
        msg = C.create_string_buffer(128)
        rc = Q().dpq_next(self.h, timeout, C.byref(ticket), _p(proof), C.byref(plen), _p(out), C.byref(st), C.cast(msg, VP), len(msg))
        return rc, (None if rc else (ticket.value, proof[: plen.value].copy(), out, st.value, msg.value.decode()))

    def close(self):
        n = U64()
        Q().dpq_close(self.h, C.byref(n))
        return n.value


def test_tickets_count_up_in_submission_order():
    f = Fake(capacity=16, servers=1)
    try:
        assert f.submit([10]) == (OK, 0)
        assert f.submit([11, 12, 13]) == (OK, 1)
        assert f.submit([14, 15]) == (OK, 4)
        got = [f.next()[1] for _ in range(6)]
        assert [g[0] for g in got] == list(range(6)), "one server finishes in submission order"
        for t, proof, out, status, msg in got:
            assert status == 0 and msg == "" and proof[0] == 10 + t and (out == 2 * np.array([10 + t, 0, 0])).all()
    finally:
        f.close()


def test_submit_refusals():
    f = Fake(capacity=4, servers=1)
    try:
        assert f.submit([]) == (INVALID, 0) and b"no inputs" in Q().dpq_last_error()
        assert f.submit([1] * 5)[0] == INVALID and b"more inputs than the stream's capacity" in Q().dpq_last_error()
        first = U64()
        assert Q().dpq_submit(f.h, None, 1, 0, C.byref(first)) == INVALID and b"null argument" in Q().dpq_last_error()
    finally:
        f.close()


def test_submit_at_capacity_is_all_or_nothing_and_times_out():
    """capacity counts uncollected jobs; a submit that does not fit submits nothing and fails with DP_ERR_TIMEOUT after its timeout
    (0: at once); a negative timeout waits until a next makes room"""
    f = Fake(capacity=4, servers=2)
    try:
        assert f.submit([1, 2, 3]) == (OK, 0)
        t0 = time.monotonic()
        assert f.submit([4, 5], timeout=0)[0] == TIMEOUT
        assert time.monotonic() - t0 < 0.1
        assert b"no room" in Q().dpq_last_error()
        t0 = time.monotonic()
        assert f.submit([4, 5], timeout=200)[0] == TIMEOUT
        assert 0.18 < time.monotonic() - t0 < 2.0
        assert f.submit([4]) == (OK, 3), "nothing of the refused submits took a ticket or a slot"
        res = {}
        th = threading.Thread(target=lambda: res.update(r=f.submit([5, 6], timeout=-1)))
        th.start()
        time.sleep(0.2)
        assert th.is_alive(), "a negative timeout waits while there is no room"
        first_two = [f.next()[1][0] for _ in range(2)]
        th.join(5)
        assert res["r"] == (OK, 4)
        assert sorted(first_two + [f.next()[1][0] for _ in range(4)]) == list(range(6))
    finally:
        f.close()


def test_next_timeouts_and_empty_stream():
    f = Fake(capacity=4, servers=1)
    try:
        t0 = time.monotonic()
        assert f.next(-1)[0] == STATE, "an empty stream refuses at once, even with an endless wait"
        assert time.monotonic() - t0 < 0.1 and b"nothing submitted is left" in Q().dpq_last_error()
        assert f.submit([7], ms=400) == (OK, 0)
        t0 = time.monotonic()
        assert f.next(0)[0] == TIMEOUT and time.monotonic() - t0 < 0.1
        assert f.next(100)[0] == TIMEOUT and b"before the timeout" in Q().dpq_last_error()
        rc, r = f.next(-1)
        assert rc == OK and r[0] == 0 and r[1][0] == 7
        assert f.next(-1)[0] == STATE
    finally:
        f.close()


def test_failed_job_fails_alone():
    f = Fake(capacity=8, servers=2)
    try:
        assert f.submit([1, -1, 2]) == (OK, 0)
        got = {r[0]: r for r in (f.next()[1] for _ in range(3))}
        assert got[1][3] == INVALID and got[1][4] == "fake job: negative input" and got[1][1].size == 0 and (got[1][2] == 0).all()
        assert got[0][3] == 0 and got[2][3] == 0 and got[2][1][0] == 2
    finally:
        f.close()


def test_close_cancels_the_jobs_not_started():
    """one server on a 200 ms job: close cancels the four queued behind it and waits for the running one"""
    f = Fake(capacity=8, servers=1)
    assert f.submit([1] * 5, ms=200) == (OK, 0)
    deadline = time.monotonic() + 5
    while Q().dpq_started(f.h) == 0 and time.monotonic() < deadline:
        time.sleep(0.005)
    t0 = time.monotonic()
    assert f.close() == 4
    assert time.monotonic() - t0 > 0.1, "close returned before the running job finished"
    f2 = Fake(capacity=8, servers=2)
    assert f2.submit([1, 2]) == (OK, 0)
    assert f2.next()[0] == OK
    time.sleep(0.05)
    assert f2.close() == 0, "finished and uncollected jobs are not cancelled"


def test_close_wakes_waiting_callers():
    f = Fake(capacity=1, servers=1)
    assert f.submit([1], ms=300) == (OK, 0)
    res = {}
    th = [threading.Thread(target=lambda: res.update(s=f.submit([2], timeout=-1))),
          threading.Thread(target=lambda: res.update(n=f.next(-1)[0]))]
    for t in th:
        t.start()
    time.sleep(0.05)
    f.close()
    for t in th:
        t.join(5)
    assert res["s"][0] == STATE and res["n"] in (OK, STATE)


def test_backlog_is_the_queue_length_when_taken():
    f = Fake(capacity=8, servers=1)
    try:
        assert f.submit([1, 2, 3, 4], ms=20) == (OK, 0)
        backlog = [f.next()[1][1][1] for _ in range(4)]
        assert backlog[1:] == [3, 2, 1] and backlog[0] in (4, 1), backlog
        assert f.submit([5]) == (OK, 4) and f.next()[1][1][1] == 1, "a lone job on an idle stream sees a backlog of 1"
    finally:
        f.close()


def test_concurrent_next_callers_get_each_result_once():
    n, callers = 400, 6
    f = Fake(capacity=n, servers=4)
    try:
        assert f.submit(list(range(n))) == (OK, 0)
        got, lock = [], threading.Lock()

        def collect():
            while True:
                rc, r = f.next(-1)
                if rc == STATE:
                    return
                assert rc == OK
                with lock:
                    got.append(r[0])
        th = [threading.Thread(target=collect) for _ in range(callers)]
        for t in th:
            t.start()
        for t in th:
            t.join(30)
        assert sorted(got) == list(range(n))
    finally:
        f.close()


def test_racing_submit_and_next_lose_nothing():
    """two threads submit in batches of 1 to 5 with an endless wait while two others collect: every ticket comes back once, with its
    own input"""
    per, cap = 300, 16
    f = Fake(capacity=cap, servers=3)
    try:
        values, lock, got = {}, threading.Lock(), []

        def produce(seed):
            rng = np.random.Generator(np.random.PCG64(seed))
            k = 0
            while k < per:
                m = int(min(rng.integers(1, 6), per - k))
                vals = [seed * 10000 + k + i for i in range(m)]
                rc, first = f.submit(vals, timeout=-1)
                assert rc == OK
                with lock:
                    values.update({first + i: v for i, v in enumerate(vals)})
                k += m

        def consume(total):
            while True:
                with lock:
                    if len(got) >= total:
                        return
                rc, r = f.next(20)
                if rc == OK:
                    with lock:
                        got.append((r[0], int(r[1][0])))
                else:
                    assert rc in (TIMEOUT, STATE)
        th = [threading.Thread(target=produce, args=(s,)) for s in (1, 2)] + [threading.Thread(target=consume, args=(2 * per,)) for _ in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join(60)
        assert sorted(t for t, _ in got) == list(range(2 * per))
        assert all(values[t] == v for t, v in got)
    finally:
        f.close()
