"""CPU tests of the batch-proving entry points (dph_zkml_prove_batch, dph_zkml_output_len, dph_zkml_trace_output,
dph_zkml_job_error): their argument refusals, and the checker's model IO that the GPU tests compare the device against."""
import ctypes as C
import numpy as np
import pytest
import dpb200
import models
import oracle_model_io as M


def _batch(handle=None, n=2, inputs=True, proofs=True, status=True, stride=64):
    x = np.zeros((max(n, 1), 8), dtype=np.int64)
    pr = np.zeros(max(n, 1) * stride, dtype=np.uint64)
    lens = np.zeros(max(n, 1), dtype=np.uint64)
    outs = np.zeros((max(n, 1), 8), dtype=np.int64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    p = lambda a, keep: a.ctypes.data_as(C.c_void_p) if keep else None
    return dpb200.host().dph_zkml_prove_batch(handle, 0, 2, p(x, inputs), n, b"m2vec", p(pr, proofs), stride, p(lens, True),
                                              p(outs, True), p(st, status), None)


@pytest.mark.parametrize("case", ["n0", "inputs", "proofs", "status"])
def test_batch_refuses_bad_arguments(case):
    """n == 0 and null inputs / proofs / status are call-level refusals, checked before anything else"""
    kw = {"n0": dict(n=0), "inputs": dict(inputs=False), "proofs": dict(proofs=False), "status": dict(status=False)}[case]
    assert _batch(**kw) == dpb200.DP_ERR_INVALID
    msg = dpb200.host().dph_last_error().decode()
    assert "dph_zkml_prove_batch" in msg and ("no inputs" in msg if case == "n0" else "null argument" in msg)


def test_batch_entry_points_without_a_device():
    """no model context can exist without a device, and a batch call without one is refused with DP_ERR_NO_DEVICE"""
    if dpb200.device_count() > 0:
        pytest.skip("a device is visible: the GPU tests cover these entry points")
    H = dpb200.host()
    desc, data, x = models.token_mlp(seed=11, tokens=8, d_model=32, d_hidden=64)
    h = C.c_void_p()
    d = np.ascontiguousarray(desc, dtype=np.int64)
    assert H.dph_model_context_new(d.ctypes.data_as(C.c_void_p), d.shape[0], data.ctypes.data_as(C.c_void_p), x.size, C.byref(h)) == dpb200.DP_ERR_NO_DEVICE
    assert _batch() == dpb200.DP_ERR_NO_DEVICE
    assert b"no CPU fallback" in H.dph_last_error()


def test_handle_entry_points_refuse_a_null_handle():
    H = dpb200.host()
    n = C.c_uint64()
    out = np.zeros(16, dtype=np.int64)
    assert H.dph_zkml_output_len(None, C.byref(n)) == dpb200.DP_ERR_INVALID
    assert H.dph_zkml_trace_output(None, out.ctypes.data_as(C.c_void_p), out.size, C.byref(n)) == dpb200.DP_ERR_INVALID
    assert H.dph_zkml_job_error(None, 0) is None


def _models():
    desc, data, x, _ = models.cnn_small(seed=3)
    yield "cnn_small", desc, data, x
    desc, data, x = models.token_mlp(seed=11, tokens=8, d_model=32, d_hidden=64)
    yield "token_mlp", desc, data, x


@pytest.mark.parametrize("name", ["cnn_small", "token_mlp"])
def test_checker_verifies_the_given_output(name):
    """model_verify_output accepts the model's true output and rejects it with one element changed"""
    desc, data, x = next((d, w, x) for n, d, w, x in _models() if n == name)
    y = M.model_output(desc, data, x)
    assert y.size == {"cnn_small": 16, "token_mlp": 8 * 32}[name]
    assert M.model_verify_output(desc, data, x, y) is None
    for k in (0, y.size - 1):
        bad = y.copy()
        bad[k] += 1
        assert M.model_verify_output(desc, data, x, bad) is not None, "%s: output element %d changed and still accepted" % (name, k)


def test_checker_refuses_an_input_outside_its_tables():
    """scaling an MLP input far out of the quantised range makes the checker's own inference refuse it (what the GPU failure-isolation
    test relies on)"""
    desc, data, x = _mlp()
    assert M.model_output(desc, data, x).size == 64
    with pytest.raises(RuntimeError, match="requantisation"):
        M.model_output(desc, data, x * 4096)


def _mlp():
    import oracle_py as O
    w, b, rq = O.synthetic_mlp(2, 64, 5)
    desc = np.zeros((6, 9), dtype=np.int64)
    desc[0::3, 1:3] = 64
    desc[1::3, 0], desc[1::3, 1:5] = 1, rq
    desc[2::3, 0] = 2
    data = np.concatenate([w.reshape(2, -1), b.reshape(2, -1)], axis=1).reshape(-1)
    return desc, data, O.synthetic_input(64, 6)
