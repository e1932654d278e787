"""ctypes view of tests/libdp_oracle_model_io.so -- TEST INFRASTRUCTURE.  The public IO of a model proof on the CPU checker:
the model's output, and the restated verifier run against an output the caller supplies.  Models are layer descriptors
(deep-prove_b200/models.py) as oracle_py.model_prove takes them; the hasher is the one oracle_py.set_hash_mode selected."""
import ctypes as C
import os
import numpy as np

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libdp_oracle_model_io.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError("checker model IO not built: run `make oracle`")
        _lib = C.CDLL(_PATH)
        _lib.dpo_io_last_error.restype = C.c_char_p
    return _lib


def _i64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.int64))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _model(desc, data, x):
    d = _i64(desc).reshape(-1, 9)
    return d, _i64(data), _i64(x).reshape(-1)


def model_output(desc, data, x):
    """zk_run(model, x).back(): the model's output in the padded layout (int64); raises when the checker refuses the input"""
    d, w, xi = _model(desc, data, x)
    args = [_ptr(d), C.c_uint32(d.shape[0]), _ptr(w), _ptr(xi), C.c_uint64(xi.size)]
    n = C.c_uint64()
    if lib().dpo_model_output(*args, None, C.c_uint64(0), C.byref(n)):
        raise RuntimeError(lib().dpo_io_last_error().decode())
    out = np.zeros(n.value, dtype=np.int64)
    if lib().dpo_model_output(*args, _ptr(out), C.c_uint64(out.size), C.byref(n)):
        raise RuntimeError(lib().dpo_io_last_error().decode())
    return out


def model_verify_output(desc, data, x, output, label=b"m2vec"):
    """prove x on the checker, then verify on a fresh transcript with `output` as the public output: None = accepted, else the
    reason"""
    d, w, xi = _model(desc, data, x)
    y = _i64(output).reshape(-1)
    rc = lib().dpo_model_verify_output(_ptr(d), C.c_uint32(d.shape[0]), _ptr(w), _ptr(xi), C.c_uint64(xi.size), _ptr(y), C.c_uint64(y.size), label)
    return None if rc == 0 else lib().dpo_io_last_error().decode()
