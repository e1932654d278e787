"""The flat-output rule of the host library's entry points (host/capi.cpp put_flat): *out_len always reports the words the output
needs; a caller buffer one word short is refused with DP_ERR_INVALID and "<entry>: output buffer too small", and a buffer of exactly
that length receives the same words the Python wrapper returns."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_py as O

pytestmark = pytest.mark.gpu
LABEL = b"m2vec"


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _short_then_exact(gpu, entry, call, exp):
    """call(out, cap, out_len) -> return code, run with cap = len(exp) - 1 and then len(exp); the short call must not write `out`"""
    n = exp.size
    short, n_short = np.zeros(n - 1, dtype=np.uint64), C.c_uint64()
    assert call(_p(short), n - 1, C.byref(n_short)) == gpu.DP_ERR_INVALID, entry
    assert gpu.host().dph_last_error().decode() == entry + ": output buffer too small"
    assert n_short.value == n and not short.any(), entry
    out, n_exact = np.zeros(n, dtype=np.uint64), C.c_uint64()
    gpu.hcheck(call(_p(out), n, C.byref(n_exact)))
    assert n_exact.value == n and (out == exp).all(), entry


def test_pcs_open(gpu):
    m = gpu.Mle.upload(O.splitmix_f(1, 1 << 10), False)
    pt = gpu._u64(O.splitmix_e(2, 10)).reshape(-1)
    _, exp = gpu.pcs_open(m, 10, pt)
    root = np.zeros(4, dtype=np.uint64)
    _short_then_exact(gpu, "dph_pcs_open", lambda *o: gpu.host().dph_pcs_open(m.h, 10, _p(pt), LABEL, *o, _p(root)), exp)


def test_pcs_batch_open_evals(gpu):
    ms = [gpu.Mle.upload(O.splitmix_f(3, 1 << 9), False), gpu.Mle.upload(O.splitmix_e(4, 1 << 8), True)]
    points = [O.splitmix_e(5, 9), O.splitmix_e(6, 8)]
    exp = gpu.pcs_batch_open_evals(ms, 10, points, [0, 1], [0, 1])
    pts = np.concatenate([gpu._u64(x).reshape(-1) for x in points])
    pnv, idx = np.array([9, 8], dtype=np.uint32), np.array([0, 1], dtype=np.uint32)
    _short_then_exact(gpu, "dph_pcs_batch_open_evals", lambda *o: gpu.host().dph_pcs_batch_open_evals(
        gpu.handles(ms), 2, 10, _p(pts), _p(pnv), 2, _p(idx), _p(idx), 2, LABEL, *o), exp)


def test_pcs_simple_batch(gpu):
    ms = [gpu.Mle.upload(O.splitmix_f(7 + i, 1 << 9), False) for i in range(3)]
    pt = gpu._u64(O.splitmix_e(10, 9)).reshape(-1)
    ev = np.concatenate([m.evaluate(pt) for m in ms])
    _, exp = gpu.pcs_simple_batch(ms, 10, pt, ev)
    root = np.zeros(4, dtype=np.uint64)
    _short_then_exact(gpu, "dph_pcs_simple_batch", lambda *o: gpu.host().dph_pcs_simple_batch(
        gpu.handles(ms), 3, 10, _p(pt), 9, _p(ev), LABEL, _p(root), *o), exp)


def test_zkml_prove(gpu):
    w, b, rq = O.synthetic_mlp(2, 64, 5)
    x = O.synthetic_input(64, 6)
    ctx = gpu.ZkmlContext(2, 64, w, b, rq)
    try:
        exp = ctx.prove(x)
        _short_then_exact(gpu, "dph_zkml_prove", lambda *o: gpu.host().dph_zkml_prove(ctx.h, _p(x), 0, LABEL, *o), exp)
    finally:
        ctx.free()


def test_conv_prove(gpu):
    filt, bias, x, uo = O.synthetic_conv(2, 2, 8, 4, 2, 3, 2, 7, 35, 36)
    _, _, exp = gpu.conv_prove(filt, bias, uo, x)
    kw, kx, rn, _ = filt.shape
    after, cleared = np.zeros((kw, 8, 8), dtype=np.int64), np.zeros((kw, 8, 8), dtype=np.int64)
    filt, bias, x = (np.ascontiguousarray(a, dtype=np.int64) for a in (filt, bias, x))
    uo = np.ascontiguousarray(uo, dtype=np.uint32)
    _short_then_exact(gpu, "dph_conv_prove", lambda *o: gpu.host().dph_conv_prove(
        kw, kx, 8, rn, _p(filt), _p(bias), _p(uo), _p(x), LABEL, _p(after), _p(cleared), *o), exp)


def test_logup_prove(gpu):
    """no Python wrapper: the exact-cap call must equal a call into an ample buffer"""
    cols = [gpu.Mle.upload(O.splitmix_f(20 + k, 1 << 6), False) for k in range(2)]
    cc, sc = np.array(O.splitmix_f(91, 2), dtype=np.uint64), np.array(O.splitmix_f(92, 2), dtype=np.uint64)

    def call(out, cap, out_len):
        return gpu.host().dph_logup_prove(gpu.handles(cols), 2, None, 1, _p(cc), _p(sc), LABEL, out, cap, out_len)
    exp = gpu.flat_out(1 << 16, call)
    _short_then_exact(gpu, "dph_logup_prove", call, exp)


def test_pcs_open_sharded(gpu):
    """world 2 over one process's mailbox, one thread (and library context) per rank; both ranks get the short cap"""
    import multigpu as mg
    nv, world = 14, 2
    ev, pt = O.splitmix_f(40, 1 << nv), gpu._u64(O.splitmix_e(41, nv)).reshape(-1)
    _, exp = gpu.pcs_open(gpu.Mle.upload(ev, False), nv, pt)
    box = mg.LocalMailbox()
    err = []

    def rank_main(r):
        try:
            gpu.init(0)
            m, v = gpu.Mle.upload(ev, False), box.for_rank()
            root = np.zeros(4, dtype=np.uint64)
            _short_then_exact(gpu, "dph_pcs_open_sharded", lambda *o: gpu.host().dph_pcs_open_sharded(
                world, r, m.h, nv, _p(pt), LABEL, C.c_void_p(v.addr), C.byref(v.seq), None, None, *o, _p(root), None), exp)
        except BaseException as e:      # surfaced below
            err.append((r, repr(e)))
    th = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not err, err
