"""The library's wait service (csrc/context.cu dp_wait_flag; DESIGN.md section 5.1) without a device: in blocking mode a waiting thread
registers its word with the poller thread and sleeps on a futex -- it must wake promptly when the word flips, burn (almost) no CPU while
it waits, time out cleanly, and many waiters must be served at once; in spin mode the same call spins."""
import ctypes as C
import threading
import time

import pytest

import dpb200


def _wait(lib, word, want, timeout, out, k):
    c0 = time.thread_time()
    t0 = time.perf_counter()
    out[k] = (lib.dp_debug_wait_flag(C.byref(word), C.c_uint64(want), C.c_double(timeout)), time.perf_counter() - t0, time.thread_time() - c0)


@pytest.fixture
def lib():
    L = dpb200.lib()
    before = L.dp_get_wait_mode()
    yield L
    L.dp_set_wait_mode(before)


def test_blocking_wait_wakes_and_sleeps(lib):
    assert lib.dp_set_wait_mode(1) == 0
    words = [C.c_uint64(0) for _ in range(12)]
    out = [None] * 12
    th = [threading.Thread(target=_wait, args=(lib, words[k], 7 + k, 5.0, out, k)) for k in range(12)]
    for t in th:
        t.start()
    time.sleep(0.25)
    for k in range(12):
        words[k].value = 7 + k
    for t in th:
        t.join()
    for k in range(12):
        seen, wall, cpu = out[k]
        assert seen == 7 + k
        assert 0.2 < wall < 1.0
        assert cpu < 0.05, "a sleeping waiter burnt %.3f s of CPU in %.3f s" % (cpu, wall)


def test_blocking_wait_times_out(lib):
    assert lib.dp_set_wait_mode(1) == 0
    w = C.c_uint64(0); out = [None]
    _wait(lib, w, 1, 0.2, out, 0)
    assert out[0][0] == (1 << 64) - 3 and 0.15 < out[0][1] < 1.0          # DP_WAIT_TIMEOUT
    w.value = 1
    _wait(lib, w, 1, 0.2, out, 0)                                          # the slot is usable again; an already-set word returns at once
    assert out[0][0] == 1 and out[0][1] < 0.05


def test_spin_mode_same_result(lib):
    assert lib.dp_set_wait_mode(0) == 0
    w = C.c_uint64(0); out = [None]
    t = threading.Thread(target=_wait, args=(lib, w, 5, 5.0, out, 0))
    t.start(); time.sleep(0.05); w.value = 5; t.join()
    assert out[0][0] == 5 and out[0][1] < 1.0
