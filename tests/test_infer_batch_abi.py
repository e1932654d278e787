"""CPU tests of the batch-inference entry point (dph_zkml_infer_batch) and of the device plan calls (dp_infer_*): argument refusals,
checked before anything else, and the refusals without a device."""
import ctypes as C
import numpy as np
import pytest
import dpb200


def _infer(handle=None, n=2, inputs=True, outputs=True, status=True):
    x = np.zeros((max(n, 1), 8), dtype=np.int64)
    y = np.zeros((max(n, 1), 8), dtype=np.int64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    p = lambda a, keep: a.ctypes.data_as(C.c_void_p) if keep else None
    return dpb200.host().dph_zkml_infer_batch(handle, p(x, inputs), n, p(y, outputs), p(st, status), None)


@pytest.mark.parametrize("case", ["n0", "inputs", "outputs", "status"])
def test_infer_refuses_bad_arguments(case):
    """n == 0 and null inputs / outputs / status are call-level refusals, checked before the device and the handle"""
    kw = {"n0": dict(n=0), "inputs": dict(inputs=False), "outputs": dict(outputs=False), "status": dict(status=False)}[case]
    assert _infer(**kw) == dpb200.DP_ERR_INVALID
    msg = dpb200.host().dph_last_error().decode()
    assert "dph_zkml_infer_batch" in msg and ("no inputs" in msg if case == "n0" else "null argument" in msg)


def test_infer_without_a_device():
    """without a device the call is refused with DP_ERR_NO_DEVICE (no CPU fallback), and so are the device plan calls"""
    if dpb200.device_count() > 0:
        pytest.skip("a device is visible: the GPU tests cover the entry point")
    assert _infer() == dpb200.DP_ERR_NO_DEVICE
    assert b"no CPU fallback" in dpb200.host().dph_last_error()
    L = dpb200.lib()
    plan = C.c_void_p()
    assert L.dp_infer_plan(None, 0, 8, C.byref(plan)) == dpb200.DP_ERR_NO_DEVICE
    assert L.dp_infer_run(None, None, 1, None, None) == dpb200.DP_ERR_NO_DEVICE
    assert L.dp_infer_free(None) == dpb200.DP_OK


def test_job_error_of_a_null_handle():
    assert dpb200.host().dph_zkml_job_error(None, 0) is None
