"""ctypes view of the product: libdeepprove_b200.so (C ABI, include/deepprove_b200.h) and
libdeepprove_host.so (C++ host mirror of the reference crates).  Plumbing for tests/bench only --
a Rust host binds the same C ABI directly (INTEGRATION.md).  Never imports anything from oracle/.
Fails loudly when the CUDA library is missing: there is no CPU fallback.
"""
import collections
import contextlib
import ctypes as C
import math
import os
import threading
import time
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdeepprove_b200.so")
HOST_LIB_PATH = os.path.join(_HERE, "libdeepprove_host.so")

P = 0xFFFFFFFF00000001
DP_OK, DP_ERR_INVALID, DP_ERR_CUDA, DP_ERR_NO_DEVICE, DP_ERR_STATE, DP_ERR_UNSUPPORTED, DP_ERR_TIMEOUT = range(7)

# Every entry point's C signature, applied once when lib() / host() load the library.  One rule: every pointer, handle, array,
# out-parameter and callback is VP; a C string is STR; restype is given for every return (INT for `int`, None for `void`).
VP, STR, U64, I64, U32, INT, F64 = C.c_void_p, C.c_char_p, C.c_uint64, C.c_int64, C.c_uint32, C.c_int, C.c_double
SIGNATURES = {
    # ---- libdeepprove_b200.so: include/deepprove_b200.h ----
    "dp_init": (INT, [INT]),
    "dp_shutdown": (INT, []),
    "dp_device_count": (INT, []),
    "dp_last_error": (STR, []),
    "dp_version": (STR, []),
    "dp_set_stream": (INT, [VP]),
    "dp_synchronize": (INT, []),
    "dp_kernel_launches": (U64, []),
    "dp_host_waits": (U64, []),
    "dp_set_wait_mode": (INT, [INT]),
    "dp_get_wait_mode": (INT, []),
    "dp_profile_enable": (INT, [INT]),
    "dp_profile_reset": (INT, []),
    "dp_profile_read_ex": (INT, [VP, VP, VP, VP, VP, INT]),
    "dp_profile_flush": (INT, []),
    "dp_mle_upload": (INT, [VP, U64, INT, VP]),
    "dp_mle_wrap_device": (INT, [VP, U64, INT, VP]),
    "dp_mle_clone": (INT, [VP, VP]),
    "dp_mle_download": (INT, [VP, VP]),
    "dp_mle_info": (INT, [VP, VP, VP, VP]),
    "dp_mle_device_ptr": (VP, [VP]),
    "dp_mle_free": (INT, [VP]),
    "dp_mle_fix_high": (INT, [VP, VP, U32]),
    "dp_mle_fix_high_new": (INT, [VP, VP, U32, VP]),
    "dp_mle_fix_low": (INT, [VP, VP, U32, VP]),
    "dp_mle_evaluate": (INT, [VP, VP, U32, VP]),
    "dp_mle_evaluate_many": (INT, [VP, U32, VP, U32, VP]),
    "dp_eq_build": (INT, [VP, U32, VP]),
    "dp_sc_create": (INT, [VP, U32, VP, U32, U32, U32, VP]),
    "dp_sc_round": (INT, [VP, VP, VP]),
    "dp_sc_set_resident_tail": (INT, [VP, INT]),
    "dp_sc_tail_fs_next": (INT, [VP, VP]),
    "dp_sc_run_tail_fs": (INT, [VP, VP, VP, VP, VP, VP]),
    "dp_sc_run_tail_fs_blake": (INT, [VP, VP, VP, VP, VP, VP]),
    "dp_sc_finish": (INT, [VP, VP, VP]),
    "dp_sc_destroy": (INT, [VP]),
    "dp_sc_current_mle": (INT, [VP, U32, VP]),
    "dp_logup_build": (INT, [VP, U32, VP, VP, VP, VP]),
    "dp_logup_num_vars": (INT, [VP, VP]),
    "dp_logup_outputs": (INT, [VP, VP]),
    "dp_logup_layer_mles": (INT, [VP, U32, VP, VP]),
    "dp_logup_free": (INT, [VP]),
    "dp_logup_layers_fs_next": (INT, [VP, U32, U32, VP]),
    "dp_logup_run_layers_fs": (INT, [VP, U32, U32, U32, VP, VP, VP, VP, VP, VP, VP, VP]),
    "dp_logup_run_layers_fs_blake": (INT, [VP, U32, U32, U32, VP, VP, VP, VP, VP, VP, VP, VP]),
    "dp_mle_linear_combination": (INT, [VP, VP, U32, VP]),
    "dp_fft_rows": (INT, [VP, U32, INT]),
    "dp_fft_rows_long": (INT, [VP, U32, INT]),
    "dp_pad_rows": (INT, [VP, U64, U32, U32, U64, VP]),
    "dp_conv_prod": (INT, [VP, VP, U32, U32, U64, VP]),
    "dp_conv_output_elements": (INT, [VP, U32, U32, VP, VP]),
    "dp_conv_output": (INT, [VP, U32, U32, VP, VP, VP, VP]),
    "dp_reverse_rows": (INT, [VP, U64, VP]),
    "dp_phi_g_init": (INT, [VP, U32, VP, INT, VP, VP]),
    "dp_phi_g_init_long": (INT, [VP, U32, VP, INT, VP, VP]),
    "dp_phi_level": (INT, [U32, U32, U32, VP, VP, INT, VP]),
    "dp_mle_repeat": (INT, [VP, U32, VP]),
    "dp_set_merkle_hasher": (INT, [INT]),
    "dp_get_merkle_hasher": (INT, []),
    "dp_poseidon2_init": (INT, [VP, VP, VP]),
    "dp_pcs_commit": (INT, [VP, U32, VP]),
    "dp_pcs_commit_many": (INT, [VP, U32, U32, VP]),
    "dp_pcs_batch_commit": (INT, [VP, U32, U32, VP]),
    "dp_pcs_comm_num_polys": (U32, [VP]),
    "dp_pcs_comm_part": (INT, [VP, U32, VP]),
    "dp_pcs_comm_info": (INT, [VP, VP, VP, VP, VP]),
    "dp_pcs_comm_codeword": (INT, [VP, VP]),
    "dp_pcs_comm_bh_evals": (INT, [VP, VP]),
    "dp_pcs_comm_free": (INT, [VP]),
    "dp_pcs_open_begin": (INT, [VP, VP, U32, VP, U32, VP, VP]),
    "dp_pcs_open_round": (INT, [VP, VP, VP, VP, VP]),
    "dp_pcs_open_final_message": (INT, [VP, VP]),
    "dp_pcs_open_query_words": (U64, [VP]),
    "dp_pcs_open_query": (INT, [VP, VP, U32, VP]),
    "dp_pcs_open_free": (INT, [VP]),
    "dp_pcs_commit_shard": (INT, [VP, U32, U32, U32, VP]),
    "dp_pcs_comm_shard_info": (INT, [VP, VP, VP, VP]),
    "dp_pcs_comm_set_shard_roots": (INT, [VP, VP, VP]),
    "dp_pcs_open_set_shard_roots": (INT, [VP, VP, VP]),
    "dp_wit_begin": (INT, [U32, VP, VP, VP]),
    "dp_wit_dense": (INT, [VP, VP, VP, U32, U32, VP]),
    "dp_wit_matmul": (INT, [VP, VP, VP, U32, U32, U32, INT, VP]),
    "dp_wit_requant": (INT, [VP, VP, U32, I64, U32, U32, U32, VP, U32]),
    "dp_wit_relu": (INT, [VP, VP, U32, VP]),
    "dp_wit_pool": (INT, [VP, VP, U32, U32, U32, U32, VP]),
    "dp_wit_finish": (INT, [VP, VP, VP]),
    "dp_wit_free": (INT, [VP]),
    "dp_infer_plan": (INT, [VP, U32, U64, VP]),
    "dp_infer_run": (INT, [VP, VP, U32, VP, VP]),
    "dp_infer_free": (INT, [VP]),
    # test hook of libdeepprove_b200.so, not part of the ABI (csrc/context.cu)
    "dp_debug_wait_flag": (U64, [VP, U64, F64]),
    # ---- libdeepprove_host.so: host/capi.cpp ----
    "dph_last_error": (STR, []),
    "dph_poseidon2_permute": (None, [VP]),
    "dph_poseidon2_selfcheck": (U64, [U64, U64]),
    "dph_set_hasher": (INT, [INT]),
    "dph_transcript_new": (VP, [STR]),
    "dph_transcript_free": (None, [VP]),
    "dph_transcript_append_f": (None, [VP, VP, U64]),
    "dph_transcript_append_msg": (None, [VP, VP, U64]),
    "dph_transcript_append_e": (None, [VP, VP, U64]),
    "dph_transcript_challenge": (None, [VP, STR, VP]),
    "dph_transcript_save_state": (None, [VP, VP, VP]),
    "dph_transcript_load_state": (INT, [VP, INT, VP]),
    "dph_sumcheck_prove_parallel": (INT, [VP, U32, VP, U32, U32, STR, VP, VP, VP, VP, VP]),
    "dph_pcs_open": (INT, [VP, U32, VP, STR, VP, U64, VP, VP]),
    "dph_zkml_context_free": (None, [VP]),
    "dph_zkml_prove": (INT, [VP, VP, INT, STR, VP, U64, VP]),
    "dph_zkml_pool_free": (None, [VP]),
    "dph_zkml_prove_concurrent": (INT, [VP, INT, U32, U32, INT, STR, VP, VP, U64, VP]),
    "dph_zkml_prove_concurrent_all": (INT, [VP, INT, U32, U32, INT, STR, VP, VP, U64, VP, VP]),
    "dph_zkml_output_len": (INT, [VP, VP]),
    "dph_zkml_trace_output": (INT, [VP, VP, U64, VP]),
    "dph_zkml_prove_batch": (INT, [VP, INT, U32, VP, U32, STR, VP, U64, VP, VP, VP, VP]),
    "dph_zkml_job_error": (STR, [VP, U32]),
    "dph_zkml_infer_batch": (INT, [VP, VP, U32, VP, VP, VP]),
    "dph_zkml_stream_open": (INT, [VP, INT, U32, STR, U64, U32, VP]),
    "dph_zkml_stream_submit": (INT, [VP, VP, U32, I64, VP]),
    "dph_zkml_stream_next": (INT, [VP, I64, VP, VP, VP, VP, VP, VP, U64]),
    "dph_zkml_stream_close": (INT, [VP, VP]),
    "dph_shm_mailbox_bytes": (U64, []),
    "dph_shm_allgather": (INT, [VP, U32, U32, VP, VP, U64, VP]),
    "dph_sumcheck_prove_sharded": (INT, [U32, U32, VP, U32, VP, U32, U32, STR, VP, VP, VP, VP, VP, VP, VP]),
    "dph_pcs_open_sharded": (INT, [U32, U32, VP, U32, VP, STR, VP, VP, VP, VP, VP, U64, VP, VP, VP]),
    "dph_sumcheck_prove_batch_polys": (INT, [U32, VP, U32, VP, U32, U32, STR, VP, VP, VP]),
    "dph_conv_prove": (INT, [U32, U32, U32, U32, VP, VP, VP, VP, STR, VP, VP, VP, U64, VP]),
    "dph_model_context_new": (INT, [VP, U32, VP, U64, VP]),
    "dph_pcs_simple_batch": (INT, [VP, U32, U32, VP, U32, VP, STR, VP, VP, U64, VP]),
    "dph_pcs_batch_open_evals": (INT, [VP, U32, U32, VP, VP, U32, VP, VP, U32, STR, VP, U64, VP]),
    "dph_logup_prove": (INT, [VP, U32, VP, U32, VP, VP, STR, VP, U64, VP]),
}
TEST_HOOKS = {"dp_debug_wait_flag"}
# every symbol include/deepprove_b200.h declares (tests check the .so exports each one)
ABI_SYMBOLS = sorted(n for n in SIGNATURES if n.startswith("dp_") and n not in TEST_HOOKS)


# must be in the environment before CUDA initialises (see dp_init): 32 hardware work queues instead of 8
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")


class DpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("deepprove_b200 error %d: %s" % (code, msg))
        self.code = code


class ScProduct(C.Structure):
    _fields_ = [("coef", C.c_uint64 * 2), ("n_idx", C.c_uint32), ("idx", C.c_uint32 * 5)]


_lib = None
_host = None


def _load(path, prefix, **kw):
    h = C.CDLL(path, **kw)
    for name, (res, args) in SIGNATURES.items():
        if name.startswith(prefix):
            f = getattr(h, name)
            f.restype, f.argtypes = res, args
    return h


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("%s not built: run `make` (or __graft_entry__.build()); the CUDA extension is "
                              "mandatory, there is no CPU fallback" % LIB_PATH)
        _lib = _load(LIB_PATH, "dp_", mode=C.RTLD_GLOBAL)
    return _lib


def host():
    global _host
    if _host is None:
        lib()
        if not os.path.exists(HOST_LIB_PATH):
            raise ImportError("%s not built: run `make`" % HOST_LIB_PATH)
        _host = _load(HOST_LIB_PATH, "dph_")
    return _host


def check(rc):
    if rc != 0:
        raise DpError(rc, lib().dp_last_error().decode())


def hcheck(rc):
    if rc != 0:
        raise DpError(rc, host().dph_last_error().decode())


def init(device=0):
    check(lib().dp_init(int(device)))


def set_wait_mode(mode):
    """0 = every proving thread spins on its completion word (lowest latency); 1 = threads sleep and ONE poller thread of the
    library wakes them (many more proofs than CPUs in flight)"""
    check(lib().dp_set_wait_mode(int(mode)))


def device_count():
    return lib().dp_device_count()


def use_torch_stream():
    """Launch on torch's current CUDA stream so torch.cuda.Event brackets our kernels."""
    import torch
    check(lib().dp_set_stream(C.c_void_p(torch.cuda.current_stream().cuda_stream)))


def _u64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.uint64))


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def handles(mles):
    """the C array of the MLEs' handles (None stays a null entry); never empty, so a zero count still passes a valid pointer"""
    return (C.c_void_p * max(1, len(mles)))(*[None if m is None else m.h for m in mles])


def flat_out(cap, call):
    """call(out, cap, out_len) fills a zeroed buffer of `cap` words and reports the length it wrote: returns those words"""
    out = np.zeros(cap, dtype=np.uint64)
    n = C.c_uint64()
    hcheck(call(_ptr(out), cap, C.byref(n)))
    return out[: n.value].copy()


class Mle:
    """Device-resident DenseMultilinearExtension (handle owner)."""

    def __init__(self, handle, keepalive=None):
        self.h = C.c_void_p(handle)
        self._keep = keepalive

    @staticmethod
    def upload(evals, is_ext):
        a = _u64(evals).reshape(-1)
        n = a.size // (2 if is_ext else 1)
        h = C.c_void_p()
        check(lib().dp_mle_upload(_ptr(a), n, int(bool(is_ext)), C.byref(h)))
        return Mle(h.value)

    @staticmethod
    def wrap_torch(t, is_ext):
        """Non-owning view of a torch int64/uint64 CUDA tensor holding canonical limbs."""
        n = t.numel() // (2 if is_ext else 1)
        h = C.c_void_p()
        check(lib().dp_mle_wrap_device(C.c_void_p(t.data_ptr()), n, int(bool(is_ext)), C.byref(h)))
        return Mle(h.value, keepalive=t)

    @staticmethod
    def eq(point):
        p = _u64(point).reshape(-1)
        h = C.c_void_p()
        check(lib().dp_eq_build(_ptr(p), p.size // 2, C.byref(h)))
        return Mle(h.value)

    def info(self):
        ln, ext, nv = C.c_uint64(), C.c_int(), C.c_uint32()
        check(lib().dp_mle_info(self.h, C.byref(ln), C.byref(ext), C.byref(nv)))
        return ln.value, bool(ext.value), nv.value

    def download(self):
        ln, ext, _ = self.info()
        out = np.empty(ln * (2 if ext else 1), dtype=np.uint64)
        check(lib().dp_mle_download(self.h, _ptr(out)))
        return out.reshape(-1, 2) if ext else out

    def fix_high(self, point):
        p = _u64(point).reshape(-1)
        check(lib().dp_mle_fix_high(self.h, _ptr(p), p.size // 2))
        return self

    def fix_low(self, point):
        p = _u64(point).reshape(-1)
        h = C.c_void_p()
        check(lib().dp_mle_fix_low(self.h, _ptr(p), p.size // 2, C.byref(h)))
        return Mle(h.value)

    def evaluate(self, point):
        p = _u64(point).reshape(-1)
        out = np.zeros(2, dtype=np.uint64)
        check(lib().dp_mle_evaluate(self.h, _ptr(p), p.size // 2, _ptr(out)))
        return out

    def clone(self):
        h = C.c_void_p()
        check(lib().dp_mle_clone(self.h, C.byref(h)))
        return Mle(h.value)

    def free(self):
        if self.h:
            lib().dp_mle_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Witness:
    """dp_wit_*: quantised inference ops and lookup-witness columns on the device (one object per proof)."""

    def __init__(self, tables):
        """tables: list of (kind, size) -- kind 0 Relu, 2 Range, 3 Clamping(size)"""
        self.n = len(tables)
        k = (C.c_uint32 * self.n)(*[int(t[0]) for t in tables]); z = (C.c_uint32 * self.n)(*[int(t[1]) for t in tables])
        self.h = C.c_void_p()
        check(lib().dp_wit_begin(self.n, k, z, C.byref(self.h)))

    @staticmethod
    def dense(w, bias, x, nrows, ncols):
        h = C.c_void_p()
        check(lib().dp_wit_dense(w.h, bias.h, x.h, int(nrows), int(ncols), C.byref(h)))
        return Mle(h.value)

    def requant(self, x, shift, fpm, intermediate_bits, clamp_table, range_table):
        nc = 2 + shift // 8
        cols = (C.c_void_p * nc)()
        check(lib().dp_wit_requant(self.h, x.h, int(shift), C.c_int64(int(fpm)), int(intermediate_bits), int(clamp_table), int(range_table), cols, nc))
        return [Mle(c) for c in cols]

    def relu(self, x, relu_table):
        h = C.c_void_p()
        check(lib().dp_wit_relu(self.h, x.h, int(relu_table), C.byref(h)))
        return Mle(h.value)

    def pool(self, x, c, hh, w, range_table):
        cols = (C.c_void_p * 5)()
        check(lib().dp_wit_pool(self.h, x.h, int(c), int(hh), int(w), int(range_table), cols))
        return [Mle(v) for v in cols]

    def finish(self):
        mu = (C.c_void_p * self.n)(); bits = C.c_uint32()
        check(lib().dp_wit_finish(self.h, mu, C.byref(bits)))
        return [Mle(v) for v in mu], bits.value

    def free(self):
        if self.h:
            lib().dp_wit_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def set_hasher(kind):
    """0 = PoseidonHasher + BasicTranscript (default), 1 = BlakeHasher + BlakeTranscript (the reference's `blake` feature); process-wide"""
    hcheck(host().dph_set_hasher(int(kind)))


class Transcript:
    """DynTranscript of the C++ host mirror (host/transcript.hpp): BasicTranscript (Poseidon2 duplex sponge) or BlakeTranscript,
    whichever set_hasher selected when it was made."""

    def __init__(self, label=b"m2vec"):
        self.h = C.c_void_p(host().dph_transcript_new(label))

    def append_f(self, f):
        f = _u64(f).reshape(-1)
        host().dph_transcript_append_f(self.h, _ptr(f), f.size)

    def append_msg(self, m):
        host().dph_transcript_append_msg(self.h, bytes(m), len(m))

    def append_e(self, e):
        e = _u64(e).reshape(-1, 2)
        host().dph_transcript_append_e(self.h, _ptr(e), e.shape[0])

    def challenge(self, label):
        out = np.zeros(2, dtype=np.uint64)
        host().dph_transcript_challenge(self.h, label, _ptr(out))
        return out

    def save_state(self):
        """-> (kind, words): kind 0 no device state, 1 the 14-word Poseidon2 sponge, 2 the DP_B3T_WORDS (80) BLAKE3 hasher image"""
        kind, words = C.c_int(-1), np.zeros(80, dtype=np.uint64)
        host().dph_transcript_save_state(self.h, C.byref(kind), _ptr(words))
        return kind.value, words

    def load_state(self, kind, words):
        w = _u64(words)
        hcheck(host().dph_transcript_load_state(self.h, int(kind), _ptr(w)))

    def free(self):
        if self.h:
            host().dph_transcript_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def profile_enable(on=True):
    check(lib().dp_profile_enable(int(on)))


def profile_reset():
    check(lib().dp_profile_reset())


def profile_read(cap=96, with_units=False):
    """-> {kernel name: (launches, total_ms, algorithmic_bytes[, units])}; process-wide (all proving threads)"""
    names = ((C.c_char * 64) * cap)()
    counts = (C.c_uint64 * cap)()
    ms = (C.c_double * cap)()
    by = (C.c_uint64 * cap)()
    un = (C.c_uint64 * cap)()
    n = lib().dp_profile_read_ex(names, counts, ms, by, un, cap)
    if with_units:
        return {names[i].value.decode(): (counts[i], ms[i], by[i], un[i]) for i in range(min(n, cap))}
    return {names[i].value.decode(): (counts[i], ms[i], by[i]) for i in range(min(n, cap))}


def make_products(products):
    """products: list of (coef (c0,c1), [mle indices])"""
    arr = (ScProduct * len(products))()
    for i, (coef, idx) in enumerate(products):
        arr[i].coef[0], arr[i].coef[1] = int(coef[0]), int(coef[1])
        arr[i].n_idx = len(idx)
        for j, v in enumerate(idx[:5]):
            arr[i].idx[j] = int(v)
    return arr


class Sumcheck:
    """Round-granular device sumcheck prover (dp_sc_*)."""

    def __init__(self, mles, products, max_nv, max_deg):
        self.mles = list(mles)
        self.prods = make_products(products)
        self.max_deg = max_deg
        self.h = C.c_void_p()
        check(lib().dp_sc_create(handles(mles), len(mles), self.prods, len(products), max_nv, max_deg, C.byref(self.h)))

    def round(self, challenge=None):
        out = np.zeros(2 * (self.max_deg + 1), dtype=np.uint64)
        c = None if challenge is None else _u64(challenge)
        check(lib().dp_sc_round(self.h, None if c is None else _ptr(c), _ptr(out)))
        return out.reshape(-1, 2)

    def finish(self, challenge):
        out = np.zeros(2 * len(self.mles), dtype=np.uint64)
        c = _u64(challenge)
        check(lib().dp_sc_finish(self.h, _ptr(c), _ptr(out)))
        return out.reshape(-1, 2)

    def destroy(self):
        if self.h:
            lib().dp_sc_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


def sumcheck_prove_parallel(mles, products, max_nv, label=b"m2vec"):
    """IOPProverState::prove_parallel through the C++ host mirror (host Poseidon2 Fiat-Shamir).
    Returns (point[nv,2], msgs[nv,deg+1,2], final_evals[n_mles,2])."""
    prods = make_products(products)
    max_deg = max(len(p[1]) for p in products)
    point = np.zeros((max_nv, 2), dtype=np.uint64)
    msgs = np.zeros((max_nv, max_deg + 1, 2), dtype=np.uint64)
    fin = np.zeros((len(mles), 2), dtype=np.uint64)
    deg = C.c_uint32()
    hcheck(host().dph_sumcheck_prove_parallel(handles(mles), len(mles), prods, len(products), max_nv, label, None, _ptr(point),
                                              _ptr(msgs), _ptr(fin), C.byref(deg)))
    return point, msgs, fin


# ---- mpcs (Basefold) -------------------------------------------------------------------------------
def _pcs_setup():
    """lib(), for callers that fetch the library through this name before using the Basefold entry points; their signatures are
    in SIGNATURES like every other"""
    return lib()


class Commitment:
    """BasefoldCommitmentWithWitness on device (dp_pcs_comm)."""

    def __init__(self, mle, full_log):
        L = lib()
        self.h = C.c_void_p()
        check(L.dp_pcs_commit(mle.h, full_log, C.byref(self.h)))
        nv, b, t = C.c_uint32(), C.c_int(), C.c_int()
        self.root = np.zeros(4, dtype=np.uint64)
        check(L.dp_pcs_comm_info(self.h, C.byref(nv), C.byref(b), C.byref(t), _ptr(self.root)))
        self.num_vars, self.is_base, self.trivial = nv.value, bool(b.value), bool(t.value)

    def codeword(self):
        v = C.c_void_p()
        check(lib().dp_pcs_comm_codeword(self.h, C.byref(v)))
        return Mle(v.value).download()

    def bh_evals(self):
        v = C.c_void_p()
        check(lib().dp_pcs_comm_bh_evals(self.h, C.byref(v)))
        return Mle(v.value).download()

    def free(self):
        if self.h:
            lib().dp_pcs_comm_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def pcs_open(mle, full_log, point, label=b"m2vec", cap=1 << 24):
    """Basefold::commit + Basefold::open through the C++ host mirror; returns (root, flat proof)."""
    p = _u64(point).reshape(-1)
    root = np.zeros(4, dtype=np.uint64)
    flat = flat_out(cap, lambda *o: host().dph_pcs_open(mle.h, full_log, _ptr(p), label, *o, _ptr(root)))
    return root, flat


def pcs_batch_open(mles, full_log, points, label=b"m2vec", cap=1 << 25):
    """commit each polynomial, then Basefold::batch_open with Evaluation::new(i, i, poly_i(point_i))."""
    return pcs_batch_open_evals(mles, full_log, points, range(len(mles)), range(len(mles)), label, cap)


def pcs_batch_open_evals(mles, full_log, points, eval_poly, eval_point, label=b"m2vec", cap=1 << 25):
    """commit each polynomial, then Basefold::batch_open with an explicit evaluation list (several polynomials may share a point)"""
    p = np.concatenate([_u64(x).reshape(-1) for x in points])
    pnv = np.ascontiguousarray([_u64(x).reshape(-1, 2).shape[0] for x in points], dtype=np.uint32)
    ep = np.ascontiguousarray(eval_poly, dtype=np.uint32); eq = np.ascontiguousarray(eval_point, dtype=np.uint32)
    return flat_out(cap, lambda *o: host().dph_pcs_batch_open_evals(handles(mles), len(mles), full_log, _ptr(p), _ptr(pnv), len(pnv),
                                                                    _ptr(ep), _ptr(eq), len(ep), label, *o))


def pcs_simple_batch(mles, full_log, point=None, evals=None, label=b"m2vec", cap=1 << 24):
    """Basefold::batch_commit of same-size device MLEs (+ simple_batch_open at `point` with the claimed `evals`): (root, flat | None)"""
    H = host()
    root = np.zeros(4, dtype=np.uint64)
    if point is None:
        hcheck(H.dph_pcs_simple_batch(handles(mles), len(mles), full_log, None, 0, None, label, _ptr(root), None, 0, None))
        return root, None
    pt = _u64(point).reshape(-1); ev = _u64(evals).reshape(-1)
    flat = flat_out(cap, lambda *o: H.dph_pcs_simple_batch(handles(mles), len(mles), full_log, _ptr(pt), pt.size // 2, _ptr(ev), label,
                                                           _ptr(root), *o))
    return root, flat


# ---- zkml MLP prover (host mirror of zkml::{Context, Prover}) -----------------------------------------
class ZkmlContext:
    """Context::generate for n_layers x [Dense(width x width)+bias -> Requant -> ReLU]: weights, bias and lookup
    tables uploaded once and committed (setup).  rq: (n_layers, 4) int64 = right_shift, fp_scale,
    fixed_point_multiplier, intermediate_bit_size."""
    _stream = None      # the open ProofStream on this handle
    _holder = None      # the StackedStream that holds this handle (StackedStream._hold)
    _calls = 0          # calls on this handle's pool in progress (_pool_call)

    def __init__(self, n_layers, width, weights, bias, rq):
        self.n_layers, self.width = n_layers, width
        w = np.ascontiguousarray(weights, dtype=np.int64).reshape(n_layers, width * width)
        b = np.ascontiguousarray(bias, dtype=np.int64).reshape(n_layers, width)
        r = np.ascontiguousarray(rq, dtype=np.int64).reshape(n_layers, 4)
        desc = np.zeros((3 * n_layers, 9), dtype=np.int64)      # per layer: Dense {width, width}, Requant {rq}, ReLU
        desc[0::3, 1:3] = width
        desc[1::3, 0], desc[1::3, 1:5] = 1, r
        desc[2::3, 0] = 2
        self._new(desc, np.concatenate([w, b], axis=1), width)
        self._out = np.zeros(1 << 22, dtype=np.uint64)

    def _new(self, desc, data, input_len):
        d = np.ascontiguousarray(desc, dtype=np.int64).reshape(-1, 9)
        w = np.ascontiguousarray(data, dtype=np.int64).reshape(-1)
        self.h = C.c_void_p()
        self._mu = threading.Lock()
        self.desc, self.data, self.input_len = d, w, int(input_len)     # kept so that stacked() can derive the stacked model
        hcheck(host().dph_model_context_new(_ptr(d), d.shape[0], _ptr(w), int(input_len), C.byref(self.h)))

    @contextlib.contextmanager
    def _pool_call(self, name):
        """Brackets a call on the handle's worker pool: refused (DP_ERR_STATE) while a StackedStream holds the handle, and counted
        while it runs, so that a StackedStream opened meanwhile finds the pool busy"""
        with self._mu:
            if self._holder is not None:
                raise DpError(DP_ERR_STATE, "%s: the handle's worker pool is busy: an open stacked stream holds it" % name)
            self._calls += 1
        try:
            yield
        finally:
            with self._mu:
                self._calls -= 1

    def prove(self, x, label=b"m2vec"):
        """inference + Prover::prove + flat proof, from a host input vector (end to end)"""
        x = np.ascontiguousarray(x, dtype=np.int64)
        n = C.c_uint64()
        hcheck(host().dph_zkml_prove(self.h, _ptr(x), 0, label, _ptr(self._out), self._out.size, C.byref(n)))
        return self._out[: n.value].copy()

    def run_inference(self, x):
        x = np.ascontiguousarray(x, dtype=np.int64)
        hcheck(host().dph_zkml_prove(self.h, _ptr(x), 1, b"", None, 0, None))

    def prove_trace(self, label=b"m2vec", want_proof=False):
        """Prover::prove on the stored inference trace (what zkml/src/bin/bench.rs:390-408 times)"""
        n = C.c_uint64()
        hcheck(host().dph_zkml_prove(self.h, None, 2, label, _ptr(self._out) if want_proof else None, self._out.size, C.byref(n)))
        return self._out[: n.value].copy() if want_proof else None

    def prove_concurrent(self, n_workers, n_proofs, device=0, e2e=False, label=b"m2vec", want_proof=False):
        """n_workers persistent host threads (own stream + device arena each) prove until n_proofs are done; returns wall
        seconds, or (seconds, flat proof of the last job handed out) when want_proof.  e2e=False: Prover::prove on the stored
        trace; e2e=True: inference + prove + serialised proof per job."""
        sec, n = C.c_double(), C.c_uint64()
        out = _ptr(self._out) if want_proof else None
        with self._pool_call("prove_concurrent"):
            hcheck(host().dph_zkml_prove_concurrent(self.h, int(device), int(n_workers), int(n_proofs), int(bool(e2e)), label, C.byref(sec),
                                                    out, self._out.size, C.byref(n)))
        return (sec.value, self._out[: n.value].copy()) if want_proof else sec.value

    def prove_concurrent_all(self, n_workers, n_proofs, stride, device=0, e2e=False, label=b"m2vec"):
        """prove_concurrent, keeping every job's flat proof (dph_zkml_prove_concurrent_all).  Returns (seconds, proofs, workers):
        proofs[j] is job j's flat proof (at most `stride` words), workers[j] the index of the worker thread that proved it."""
        out = np.zeros(int(n_proofs) * int(stride), dtype=np.uint64)
        lens = np.zeros(int(n_proofs), dtype=np.uint64)
        workers = np.zeros(int(n_proofs), dtype=np.uint32)
        sec = C.c_double()
        with self._pool_call("prove_concurrent_all"):
            hcheck(host().dph_zkml_prove_concurrent_all(self.h, int(device), int(n_workers), int(n_proofs), int(bool(e2e)), label, C.byref(sec),
                                                        _ptr(out), int(stride), _ptr(lens), _ptr(workers)))
        out = out.reshape(int(n_proofs), int(stride))
        return sec.value, [out[j, : int(lens[j])] for j in range(int(n_proofs))], workers

    @property
    def output_len(self):
        """elements of the model's output: the last node's output tensor in the padded layout"""
        n = C.c_uint64()
        hcheck(host().dph_zkml_output_len(self.h, C.byref(n)))
        return n.value

    def trace_output(self):
        """the model output (int64) of the stored trace, after prove(x) or run_inference(x)"""
        out = np.zeros(self.output_len, dtype=np.int64)
        n = C.c_uint64()
        hcheck(host().dph_zkml_trace_output(self.h, _ptr(out), out.size, C.byref(n)))
        return out[: n.value].copy()

    def prove_batch(self, inputs, n_workers, device=0, label=b"m2vec", stride=None):
        """Prove n distinct inputs ([n, input_len] int64) end to end on the worker pool (dph_zkml_prove_batch).  Returns (seconds,
        proofs, outputs, status, errors): proofs[j] is input j's flat proof (empty when it failed), outputs[j] its model output
        ([n, output_len] int64), status[j] 0 or its error code, errors[j] None or its message.  The default stride is the length of
        one proof of this model (measured once, on the first input, and kept)."""
        x = np.ascontiguousarray(inputs, dtype=np.int64)
        if x.ndim != 2 or x.shape[0] == 0 or x.shape[1] != self.input_len:
            raise ValueError("prove_batch: inputs must be [n >= 1, %d]" % self.input_len)
        n = x.shape[0]
        with self._pool_call("prove_batch"):
            if stride is None:
                stride = self._default_stride(x[0], device, label)
            proofs = np.zeros((n, int(stride)), dtype=np.uint64)
            lens = np.zeros(n, dtype=np.uint64)
            outputs = np.zeros((n, self.output_len), dtype=np.int64)
            status = np.zeros(n, dtype=np.int32)
            sec = C.c_double()
            hcheck(host().dph_zkml_prove_batch(self.h, int(device), int(n_workers), _ptr(x), n, label, _ptr(proofs), int(stride), _ptr(lens),
                                               _ptr(outputs), _ptr(status), C.byref(sec)))
            errors = [None if status[j] == 0 else host().dph_zkml_job_error(self.h, j).decode() for j in range(n)]
        return sec.value, [proofs[j, : int(lens[j])] for j in range(n)], outputs, status, errors

    def _default_stride(self, x, device, label):
        """the length of one proof of this model: measured once, by proving input x, and kept"""
        if getattr(self, "_proof_words", None) is None:
            one = np.zeros(1 << 23, dtype=np.uint64)
            lens, st = np.zeros(1, dtype=np.uint64), np.zeros(1, dtype=np.int32)
            y = np.zeros(self.output_len, dtype=np.int64)
            x = np.ascontiguousarray(x, dtype=np.int64)
            hcheck(host().dph_zkml_prove_batch(self.h, int(device), 1, _ptr(x), 1, label, _ptr(one), one.size, _ptr(lens), _ptr(y),
                                               _ptr(st), None))
            if st[0] != 0:
                raise DpError(int(st[0]), "sizing the proof stride on input 0: %s" % host().dph_zkml_job_error(self.h, 0).decode())
            self._proof_words = int(lens[0])
        return self._proof_words

    def open_stream(self, n_workers, device=0, label=b"m2vec", stride=None, capacity=None):
        """A ProofStream on the handle's worker pool (dph_zkml_stream_open): submit inputs while proofs run and collect each result
        when its proof finishes.  The pool is held until the stream closes.  stride: the longest proof a job may return (default:
        prove_batch's, which proves one all-zero input the first time); capacity: jobs submitted and not yet collected (default
        4 * n_workers)."""
        with self._pool_call("open_stream"):
            if stride is None:
                stride = self._default_stride(np.zeros(self.input_len, dtype=np.int64), device, label)
            return ProofStream(self, n_workers, device, label, stride, 4 * int(n_workers) if capacity is None else capacity)

    def infer_batch(self, inputs):
        """The model's outputs for n inputs ([n, input_len] int64, each value in [-128, 127]) without proving, on the int8 tensor
        cores (dph_zkml_infer_batch): the same outputs and per-input failures as prove_batch.  Returns (seconds, outputs [n,
        output_len] int64, status, errors)."""
        with self._pool_call("infer_batch"):
            return self._infer_batch(inputs)

    def _infer_batch(self, inputs):
        """infer_batch without the _pool_call bracket: the screening of the StackedStream that holds this handle"""
        x = np.ascontiguousarray(inputs, dtype=np.int64)
        if x.ndim != 2 or x.shape[0] == 0 or x.shape[1] != self.input_len:
            raise ValueError("infer_batch: inputs must be [n >= 1, %d]" % self.input_len)
        n = x.shape[0]
        outputs = np.zeros((n, self.output_len), dtype=np.int64)
        status = np.zeros(n, dtype=np.int32)
        sec = C.c_double()
        hcheck(host().dph_zkml_infer_batch(self.h, _ptr(x), n, _ptr(outputs), _ptr(status), C.byref(sec)))
        errors = [None if status[j] == 0 else host().dph_zkml_job_error(self.h, j).decode() for j in range(n)]
        return sec.value, outputs, status, errors

    def stacked(self, rows):
        """A StackedContext that proves up to `rows` inputs of this model in one proof (models.stack_rows).  It is a model of its own,
        set up and committed on its own handle; this context stays usable and screens the stacked proofs' inputs."""
        return StackedContext(self, rows)

    def free(self):
        if self.h:
            if self._holder is not None:                       # a stacked stream proving on this handle or screening on it
                self._holder.close()
            if getattr(self, "_stream", None) is not None:     # dph_zkml_context_free closes it
                self._stream.h, self._stream = C.c_void_p(), None
            host().dph_zkml_context_free(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class StreamTimeout(DpError):
    """a ProofStream wait ran out (DP_ERR_TIMEOUT)"""


class StreamResult:
    """One finished stream job: ticket, proof (flat, empty when the job failed), output (int64, the padded layout; zeros when it
    failed), status (0 or its error code), error (None or its message) and output_float (the dequantised real output entries for a
    model made by ModelContext.from_onnx, else None)."""
    __slots__ = ("ticket", "proof", "output", "status", "error", "output_float")

    def __init__(self, ticket, proof, output, status, error, output_float):
        self.ticket, self.proof, self.output, self.status, self.error, self.output_float = ticket, proof, output, status, error, output_float


def _ms(timeout):
    """seconds (None: for ever) as the C ABI's timeout_ms"""
    return -1 if timeout is None else max(0, int(round(float(timeout) * 1000)))


class ProofStream:
    """dph_zkml_stream_*: inputs submitted while proofs run, each result collected when its proof finishes, in completion order.
    Each job is what prove_batch does for one input, except that a proof longer than the stride fails that job alone.  Made by
    ZkmlContext.open_stream; a context manager.  submit and next may be called from different threads at once."""

    def __init__(self, ctx, n_workers, device, label, stride, capacity, dequantize=True):
        self.ctx, self.stride, self.capacity = ctx, int(stride), int(capacity)
        self._output_len = ctx.output_len
        self._metadata = getattr(ctx, "metadata", None) if dequantize else None
        self.h = C.c_void_p()
        hcheck(host().dph_zkml_stream_open(ctx.h, int(device), int(n_workers), label, self.stride, self.capacity, C.byref(self.h)))
        ctx._stream = self

    def _check(self, rc):
        if rc == DP_ERR_TIMEOUT:
            raise StreamTimeout(rc, host().dph_last_error().decode())
        hcheck(rc)

    def _open(self):
        if not self.h:
            raise DpError(DP_ERR_STATE, "the stream is closed")

    def submit(self, inputs, timeout=None):
        """Queue inputs ([n, input_len] int64, or one [input_len]); all or nothing.  Waits up to `timeout` seconds (None: for ever, 0:
        not at all) for room in the capacity, else raises StreamTimeout.  Returns their tickets (uint64, consecutive)."""
        self._open()
        x = np.ascontiguousarray(inputs, dtype=np.int64)
        x = x[None] if x.ndim == 1 else x
        if x.ndim != 2 or x.shape[0] == 0 or x.shape[1] != self.ctx.input_len:
            raise ValueError("submit: inputs must be [n >= 1, %d]" % self.ctx.input_len)
        first = C.c_uint64()
        self._check(host().dph_zkml_stream_submit(self.h, _ptr(x), x.shape[0], _ms(timeout), C.byref(first)))
        return np.arange(first.value, first.value + x.shape[0], dtype=np.uint64)

    def submit_float(self, inputs, timeout=None):
        """submit on float inputs ([n, *input shape] or one [*input shape], in [-1, 1]) of a model made by ModelContext.from_onnx,
        quantised with its metadata as prove_batch_float does"""
        md = getattr(self.ctx, "metadata", None)
        if md is None:
            raise ValueError("submit_float: the context has no quantisation metadata (build it with ModelContext.from_onnx)")
        return self.submit(md.quantize_input(np.asarray(inputs, dtype=np.float32)), timeout)

    def next(self, timeout=None):
        """The next finished job as a StreamResult.  Raises StreamTimeout when none finishes within `timeout` seconds (None: for
        ever), and DpError DP_ERR_STATE at once when nothing submitted is left to collect."""
        self._open()
        proof = np.empty(self.stride, dtype=np.uint64)
        out = np.empty(self._output_len, dtype=np.int64)
        ticket, plen, st = C.c_uint64(), C.c_uint64(), C.c_int32()
        msg = C.create_string_buffer(1024)
        self._check(host().dph_zkml_stream_next(self.h, _ms(timeout), C.byref(ticket), _ptr(proof), C.byref(plen), _ptr(out), C.byref(st),
                                                C.cast(msg, C.c_void_p), len(msg)))
        md = self._metadata
        return StreamResult(ticket.value, proof[: plen.value].copy(), out, st.value, msg.value.decode() if st.value else None,
                            None if md is None else md.dequantize_output(out))

    def results(self, timeout=None):
        """Yields results until everything submitted so far has been collected"""
        while True:
            try:
                r = self.next(timeout)
            except DpError as e:
                if e.code == DP_ERR_STATE:
                    return
                raise
            yield r

    def close(self):
        """Cancel the jobs no worker has started, wait for the running ones, drop uncollected results and release the pool.
        Returns the number cancelled (0 when already closed)."""
        if not self.h:
            return 0
        n = C.c_uint64()
        hcheck(host().dph_zkml_stream_close(self.h, C.byref(n)))
        self.h, self.ctx._stream = C.c_void_p(), None
        return n.value

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class StackedResult:
    """One input's result from a StackedStream: ticket; proof (the flat proof of its group, one array shared by every input of that
    proof; empty when screened out or failed); public_output (that proof's [R][base_output_len] output matrix, padding rows included,
    shared likewise; [0][base_output_len] when screened out); proof_id (-1 when screened out); row (its row in the proof, or -1);
    output (its row of public_output; zeros when it failed); status (0 or its error code); error (None or its message); output_float
    (the dequantised real output entries for a model made by ModelContext.from_onnx, else None)."""
    __slots__ = ("ticket", "proof", "public_output", "proof_id", "row", "output", "status", "error", "output_float")

    def __init__(self, ticket, proof, public_output, proof_id, row, output, status, error, output_float):
        self.ticket, self.proof, self.public_output, self.proof_id, self.row = ticket, proof, public_output, proof_id, row
        self.output, self.status, self.error, self.output_float = output, status, error, output_float


class StackedStream:
    """Arriving inputs grouped into stacked proofs.  Made by StackedContext.open_stream; a context manager.  submit and next may be
    called from several threads at once, and each result goes to exactly one next.

    One grouping thread closes a group when `rows` inputs are pending, or when the oldest pending input has waited max_wait seconds.
    It screens the group's inputs in one screen() call (infer_batch: (seconds, outputs, status, errors)); an input that fails gets its
    result at once, with that status and message.  The survivors, in submission order, are padded to R rows with copies of the last
    (models.pad_rows) and submitted to the prover (a ProofStream of the stacked model) as one job; a group is never topped up from
    later arrivals.  open_prover(x) returns that prover; it is called once, with the first group's padded input.  A collector thread
    takes each finished job and gives every input of its group its own result.  The class touches no device itself, so that tests
    can drive it with a fake screener and prover.  screen_calls and screen_seconds count the groups screened and the seconds screen()
    reported for them."""
    POLL_S = 0.05       # the collector's longest wait inside the prover's next before it looks whether the stream is closing

    def __init__(self, rows, R, input_len, output_len, n_workers, max_wait, capacity, screen, open_prover, metadata=None, thread_init=None):
        import models
        self.rows, self.R, self.input_len, self.output_len = int(rows), int(R), int(input_len), int(output_len)
        self.max_wait, self.capacity = float(max_wait), (4 * int(n_workers) * int(rows) if capacity is None else int(capacity))
        if int(n_workers) < 1:
            raise ValueError("open_stream: n_workers must be >= 1")
        if not (math.isfinite(self.max_wait) and self.max_wait >= 0):
            raise ValueError("open_stream: max_wait must be a finite number of seconds >= 0")
        if self.capacity < self.rows:
            raise ValueError("open_stream: capacity (%d) must be at least rows (%d)" % (self.capacity, self.rows))
        self._screen, self._open_prover, self._pad, self._metadata, self._thread_init = screen, open_prover, models.pad_rows, metadata, thread_init
        self._prover = None
        self._cv = threading.Condition()
        self._pending = collections.deque()      # (ticket, input, arrival time), not yet in a group
        self._ready = collections.deque()        # results not yet collected by next
        self._groups = {}                        # proof_id -> tickets of the group's survivors, while its proof is out
        self._next_ticket = self._uncollected = self._next_proof = self._cancelled = self._jobs = 0     # _jobs: submitted, uncollected
        self._closed = False
        self._holds = ()
        self.screen_calls, self.screen_seconds = 0, 0.0
        self._threads = [threading.Thread(target=f, daemon=True) for f in (self._group_loop, self._collect_loop)]
        for t in self._threads:
            t.start()

    def _hold(self, ctxs):
        """Reserves the handles for this stream: refused (DP_ERR_STATE) when a call or a stream is on any of their pools"""
        for c in ctxs:
            c._mu.acquire()
        try:
            for c in ctxs:
                if c._holder is not None or c._stream is not None or c._calls:
                    raise DpError(DP_ERR_STATE, "open_stream: the handle's worker pool is busy with another call or stream")
            for c in ctxs:
                c._holder = self
            self._holds = tuple(ctxs)
        finally:
            for c in ctxs:
                c._mu.release()

    # ---- the grouping thread ----
    def _group_loop(self):
        while True:
            with self._cv:
                while len(self._pending) < self.rows:
                    if self._closed:
                        return
                    left = None if not self._pending else self._pending[0][2] + self.max_wait - time.monotonic()
                    if left is not None and left <= 0:
                        break
                    self._cv.wait(left)
                if self._closed:
                    return
                take = [self._pending.popleft() for _ in range(min(self.rows, len(self._pending)))]
            self._run_group(np.array([t[0] for t in take], dtype=np.uint64), np.stack([t[1] for t in take]))

    def _run_group(self, tickets, x):
        n = len(tickets)
        try:
            if self._thread_init is not None:
                self._thread_init()
                self._thread_init = None
            sec, _, status, errors = self._screen(x)
            self.screen_calls += 1
            self.screen_seconds += sec
        except Exception as e:                   # a call-level failure fails the whole group
            status, errors = np.full(n, getattr(e, "code", DP_ERR_INVALID)), [str(e)] * n
        ok = np.flatnonzero(np.asarray(status) == 0)
        self._post([self._result(tickets[j], -1, -1, None, None, int(status[j]), errors[j]) for j in range(n) if status[j] != 0])
        if ok.size == 0:
            return
        padded = self._pad(x[ok], self.R)
        with self._cv:
            if self._closed:
                self._cancelled += ok.size
                return
            pid = self._next_proof                    # the prover's tickets count up from 0 as groups are submitted: ticket == proof_id
            self._groups[pid] = tickets[ok]
            self._next_proof += 1
        try:
            if self._prover is None:
                self._prover = self._open_prover(padded)
            self._prover.submit(padded)
        except Exception as e:
            with self._cv:
                del self._groups[pid]
                self._next_proof -= 1
            code = getattr(e, "code", DP_ERR_INVALID)
            self._post([self._result(t, -1, -1, None, None, code, str(e)) for t in tickets[ok]])
            return
        with self._cv:
            self._jobs += 1
            self._cv.notify_all()

    # ---- the collector thread ----
    def _collect_loop(self):
        while True:
            with self._cv:
                self._cv.wait_for(lambda: self._closed or self._jobs > 0)
                if self._closed:                      # close() closes the prover once this thread is out of its next
                    return
            try:
                r = self._prover.next(self.POLL_S)
            except StreamTimeout:
                continue
            except Exception as e:                    # the prover failed as a whole: fail every group still out, and stop
                with self._cv:
                    lost, self._groups, self._jobs = self._groups, {}, 0
                self._post([self._result(t, -1, -1, None, None, getattr(e, "code", DP_ERR_INVALID), str(e))
                            for ts in lost.values() for t in ts])
                return
            with self._cv:
                tickets = self._groups.pop(int(r.ticket))
                self._jobs -= 1
            public = r.output.reshape(self.R, self.output_len)
            self._post([self._result(t, int(r.ticket), row, r.proof, public, r.status, r.error) for row, t in enumerate(tickets)])

    def _result(self, ticket, proof_id, row, proof, public, status, error):
        if proof is None:
            proof, public = np.zeros(0, dtype=np.uint64), np.zeros((0, self.output_len), dtype=np.int64)
        out = public[row] if row >= 0 else np.zeros(self.output_len, dtype=np.int64)
        return StackedResult(int(ticket), proof, public, proof_id, row, out, int(status), error if status else None,
                             None if self._metadata is None else self._metadata.dequantize_output(out))

    def _post(self, results):
        if results:
            with self._cv:
                self._ready.extend(results)
                self._cv.notify_all()

    # ---- the caller's side ----
    def _wait(self, deadline, what):
        left = None if deadline is None else deadline - time.monotonic()
        if left is not None and left <= 0:
            raise StreamTimeout(DP_ERR_TIMEOUT, what)
        self._cv.wait(left)

    def submit(self, inputs, timeout=None):
        """Queue inputs ([n, base_input_len] int64, or one [base_input_len]); all or nothing.  Waits up to `timeout` seconds (None: for
        ever, 0: not at all) for room in the capacity (inputs submitted and not yet collected), else raises StreamTimeout; n > capacity
        is DP_ERR_INVALID.  Returns their tickets (uint64, consecutive, counted from 0 across the stream)."""
        x = np.array(inputs, dtype=np.int64)     # a copy: the caller may reuse its buffer at once
        x = x[None] if x.ndim == 1 else x
        if x.ndim != 2 or x.shape[0] == 0 or x.shape[1] != self.input_len:
            raise ValueError("submit: inputs must be [n >= 1, %d]" % self.input_len)
        n = x.shape[0]
        if n > self.capacity:
            raise DpError(DP_ERR_INVALID, "submit: %d inputs exceed the stream's capacity of %d" % (n, self.capacity))
        deadline = None if timeout is None else time.monotonic() + max(0.0, float(timeout))
        with self._cv:
            while self._uncollected + n > self.capacity and not self._closed:
                self._wait(deadline, "submit: no room for %d inputs before the timeout" % n)
            if self._closed:
                raise DpError(DP_ERR_STATE, "the stream is closed")
            first = self._next_ticket
            self._next_ticket += n
            self._uncollected += n
            now = time.monotonic()
            self._pending.extend((first + j, x[j], now) for j in range(n))
            self._cv.notify_all()
        return np.arange(first, first + n, dtype=np.uint64)

    def submit_float(self, inputs, timeout=None):
        """submit on float inputs ([n, *input shape] or one [*input shape], in [-1, 1]) of a model made by ModelContext.from_onnx,
        quantised with the base's metadata as prove_stacked_float does"""
        if self._metadata is None:
            raise ValueError("submit_float: the base context has no quantisation metadata (build it with ModelContext.from_onnx)")
        return self.submit(self._metadata.quantize_input(np.asarray(inputs, dtype=np.float32)), timeout)

    def next(self, timeout=None):
        """One input's StackedResult, in completion order.  Raises StreamTimeout when none is ready within `timeout` seconds (None: for
        ever), and DpError DP_ERR_STATE at once when nothing submitted is left to collect."""
        deadline = None if timeout is None else time.monotonic() + max(0.0, float(timeout))
        with self._cv:
            while not self._ready:
                if self._closed:
                    raise DpError(DP_ERR_STATE, "the stream is closed")
                if self._uncollected == 0:
                    raise DpError(DP_ERR_STATE, "next: nothing submitted is left to collect")
                self._wait(deadline, "next: no result before the timeout")
            self._uncollected -= 1
            self._cv.notify_all()
            return self._ready.popleft()

    def results(self, timeout=None):
        """Yields results until everything submitted so far has been collected"""
        while True:
            try:
                r = self.next(timeout)
            except DpError as e:
                if e.code == DP_ERR_STATE:
                    return
                raise
            yield r

    def close(self):
        """Cancel the inputs not yet in a submitted group and the groups no worker has started, wait for the running proofs, drop the
        uncollected results and release both handles.  Returns the number of inputs cancelled (0 when already closed)."""
        with self._cv:
            if self._closed:
                return 0
            self._closed = True
            cancelled = len(self._pending)
            self._pending.clear()
            self._cv.notify_all()
        for t in self._threads:
            t.join()
        if self._prover is not None:
            n_jobs = self._prover.close()             # the prover starts jobs in ticket order: the cancelled ones are the last
            ids = sorted(self._groups)
            cancelled += sum(self._groups[i].size for i in ids[len(ids) - n_jobs:]) if n_jobs else 0
        self._ready.clear()
        self._groups.clear()
        for c in self._holds:
            with c._mu:
                if c._holder is self:
                    c._holder = None
        return cancelled + self._cancelled

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class ModelContext(ZkmlContext):
    """Context::generate for a general layer list (Dense / Requant / ReLU / Convolution / Maxpool2D), see
    dph_model_context_new: desc (n_nodes, 9) int64, data = weights in node order, input_len = padded input length."""

    def __init__(self, desc, data, input_len):
        self._new(desc, data, input_len)
        self._out = np.zeros(1 << 23, dtype=np.uint64)
        self.metadata = None

    @classmethod
    def from_onnx(cls, path, calibration=None):
        """import a float ONNX model (onnx_import.py: AbsoluteMax quantisation and padding as the reference's default loader does,
        or, given calibration samples [n, *input shape] in [-1, 1], the reference's InferenceObserver on them);
        .metadata quantises float inputs (quantize_input) and dequantises outputs (dequantize_output)"""
        import onnx_import
        desc, data, input_len, md, _, _ = onnx_import.import_onnx(path, calibration)
        ctx = cls(desc, data, input_len)
        ctx.metadata = md
        return ctx

    def prove_batch_float(self, inputs, n_workers, device=0, label=b"m2vec", stride=None):
        """prove_batch on float inputs ([n, *input shape] in [-1, 1]) of a model made by from_onnx: quantises each input with
        .metadata, proves them all, and returns (proofs, outputs, float_outputs, status, errors) -- outputs are the integer model
        outputs in the padded layout, float_outputs their real entries dequantised"""
        if self.metadata is None:
            raise ValueError("prove_batch_float: the context has no quantisation metadata (build it with ModelContext.from_onnx)")
        x = np.asarray(inputs, dtype=np.float32)
        x = self.metadata.quantize_input(x.reshape((-1,) + self.metadata.input_shape))
        _, proofs, outputs, status, errors = self.prove_batch(x, n_workers, device, label, stride)
        return proofs, outputs, self.metadata.dequantize_output(outputs), status, errors

    def infer_batch_float(self, inputs):
        """infer_batch on float inputs ([n, *input shape] in [-1, 1]) of a model made by from_onnx: quantises each input with
        .metadata, infers them all without proving, and returns (outputs, float_outputs, status, errors) as prove_batch_float does"""
        if self.metadata is None:
            raise ValueError("infer_batch_float: the context has no quantisation metadata (build it with ModelContext.from_onnx)")
        x = np.asarray(inputs, dtype=np.float32)
        x = self.metadata.quantize_input(x.reshape((-1,) + self.metadata.input_shape))
        _, outputs, status, errors = self.infer_batch(x)
        return outputs, self.metadata.dequantize_output(outputs), status, errors


class StackedContext(ModelContext):
    """Many inputs of one model in one proof: the base model's Dense layers as the reference's MatMul of an input matrix [R][K] by the
    constant weight matrix (models.stack_rows), with R = p2(rows) and row r of the input matrix holding one input.  The proof is an
    ordinary proof of that stacked model; its public output is the whole [R][output_len] matrix.  Made by ZkmlContext.stacked(rows);
    keeps the base context, which screens inputs before they are proved.  rows, R, base_input_len, base_output_len and the base's
    metadata (None unless made by ModelContext.from_onnx) are attributes."""

    def __init__(self, base, rows):
        import models
        desc, data, input_len, R = models.stack_rows(base.desc, base.data, base.input_len, rows)
        ModelContext.__init__(self, desc, data, input_len)
        self.base, self.rows, self.R = base, int(rows), R
        self.base_input_len, self.base_output_len = base.input_len, base.output_len
        self.metadata = getattr(base, "metadata", None)

    def prove_stacked(self, inputs, n_workers, device=0, label=b"m2vec", stride=None):
        """Prove n inputs ([n, base_input_len] int64, each value in [-128, 127]), `rows` per proof.
          1. Screen every input with the base context's infer_batch, on the calling thread (which, as for infer_batch, needs init()):
             an input it fails keeps that status and message and is not proved, since one failing row would fail every input of its
             proof.
          2. Group the others in order, `rows` per proof; the last group is padded to R rows with copies of its last input (an input
             that passed screening, so the padding cannot fail a lookup; a zero row's bias chain could).
          3. Prove each group as one input of this model with prove_batch (its worker pool, stride, refusals and wait modes).
        Returns (seconds, proofs[g], group_outputs [G, R * base_output_len] (the public output of proof g), outputs [n,
        base_output_len] (zeros where the input failed), status[n], errors[n], proof_of[n] (-1 when screened out), row_of[n]).
        seconds is the screening plus the proving time.  Should a proof fail after screening, every input of its group gets its
        status and message."""
        import models
        x = np.ascontiguousarray(inputs, dtype=np.int64)
        if x.ndim != 2 or x.shape[0] == 0 or x.shape[1] != self.base_input_len:
            raise ValueError("prove_stacked: inputs must be [n >= 1, %d]" % self.base_input_len)
        n, R, out_len = x.shape[0], self.R, self.base_output_len
        sec, _, status, errors = self.base.infer_batch(x)
        status, errors = status.copy(), list(errors)
        ok = np.flatnonzero(status == 0)
        groups = [ok[g: g + self.rows] for g in range(0, ok.size, self.rows)]
        outputs = np.zeros((n, out_len), dtype=np.int64)
        proof_of, row_of = np.full(n, -1, dtype=np.int64), np.full(n, -1, dtype=np.int64)
        if not groups:
            return sec, [], np.zeros((0, R * out_len), dtype=np.int64), outputs, status, errors, proof_of, row_of
        stacked = np.stack([models.pad_rows(x[idx], R) for idx in groups])
        prove_sec, proofs, group_outputs, gstatus, gerrors = self.prove_batch(stacked, n_workers, device, label, stride)
        for g, idx in enumerate(groups):
            proof_of[idx], row_of[idx] = g, np.arange(idx.size)
            if gstatus[g] == 0:
                outputs[idx] = group_outputs[g].reshape(R, out_len)[: idx.size]
            else:
                status[idx] = gstatus[g]
                for j in idx:
                    errors[j] = gerrors[g]
        return sec + prove_sec, proofs, group_outputs, outputs, status, errors, proof_of, row_of

    def prove_stacked_float(self, inputs, n_workers, device=0, label=b"m2vec", stride=None):
        """prove_stacked on float inputs ([n, *input shape] in [-1, 1]) of a model made by from_onnx: quantises each input with the
        base's metadata and returns (proofs, group_outputs, outputs, float_outputs, status, errors, proof_of, row_of), float_outputs
        being each input's real output entries dequantised"""
        if self.metadata is None:
            raise ValueError("prove_stacked_float: the base context has no quantisation metadata (build it with ModelContext.from_onnx)")
        x = np.asarray(inputs, dtype=np.float32)
        x = self.metadata.quantize_input(x.reshape((-1,) + self.metadata.input_shape))
        _, proofs, group_outputs, outputs, status, errors, proof_of, row_of = self.prove_stacked(x, n_workers, device, label, stride)
        return proofs, group_outputs, outputs, self.metadata.dequantize_output(outputs), status, errors, proof_of, row_of

    def open_stream(self, n_workers, max_wait, device=0, label=b"m2vec", stride=None, capacity=None):
        """A StackedStream: inputs submitted one by one are grouped, up to `rows` per proof, and proved as prove_stacked proves a group,
        on a ProofStream of this handle with n_workers workers.  A group closes when `rows` inputs are pending or when its oldest input
        has waited max_wait seconds.  Both handles are held until the stream closes: this handle's pool proves for it and the base
        context screens for it, so calls on either pool are refused (DP_ERR_STATE) meanwhile.  stride: the longest proof a job may
        return; by default the proof length this context measured before, else that of the first group's proof, measured on that
        group (screened and copy-padded) before its job is submitted.  capacity: inputs submitted and not yet collected (default 4 *
        n_workers * rows).  The calling thread needs no device; the grouping thread calls init(device) itself."""
        def open_prover(x):
            words = stride if stride is not None else self._default_stride(x, device, label)
            return ProofStream(self, n_workers, device, label, words, s.capacity, dequantize=False)   # metadata is the base's
        s = StackedStream(self.rows, self.R, self.base_input_len, self.base_output_len, n_workers, max_wait, capacity,
                          self.base._infer_batch, open_prover, self.metadata, lambda: init(device))
        try:
            s._hold((self.base, self))
            if stride is not None or getattr(self, "_proof_words", None) is not None:
                s._prover = open_prover(None)          # the stride is known: open now, so that a busy pool refuses the open itself
        except BaseException:
            s.close()
            raise
        return s


def sumcheck_prove_batch_polys(T, mles, products, max_nv, label=b"m2vec"):
    """IOPProverState::prove_batch_polys (devirgo split into T contiguous slices) through the C++ host mirror."""
    prods = make_products(products)
    max_deg = max(len(p[1]) for p in products)
    point = np.zeros((max_nv, 2), dtype=np.uint64)
    msgs = np.zeros((max_nv, max_deg + 1, 2), dtype=np.uint64)
    fin = np.zeros((len(mles), 2), dtype=np.uint64)
    hcheck(host().dph_sumcheck_prove_batch_polys(T, handles(mles), len(mles), prods, len(products), max_nv, label, _ptr(point), _ptr(msgs), _ptr(fin)))
    return point, msgs, fin


# ---- FFT-convolution layer (host/conv.hpp) -------------------------------------------------------------
def conv_prove(filt, bias, unpadded_out, x, label=b"m2vec", cap=1 << 20, prove=True):
    """Convolution::op (+ prove_convolution_step when `prove`) on a padded layer: filt [kw, kx, real_nw, real_nw],
    bias [kw], x [kx, n_x, n_x] (int64).  Returns (after_bias, cleared, flat_proof | None)."""
    filt = np.ascontiguousarray(filt, dtype=np.int64); bias = np.ascontiguousarray(bias, dtype=np.int64); x = np.ascontiguousarray(x, dtype=np.int64)
    kw, kx, rn, _ = filt.shape
    n_x = x.shape[1]
    uo = np.ascontiguousarray(unpadded_out, dtype=np.uint32)
    after = np.zeros((kw, n_x, n_x), dtype=np.int64)
    cleared = np.zeros((kw, n_x, n_x), dtype=np.int64)

    def call(out, cap, out_len):
        return host().dph_conv_prove(kw, kx, n_x, rn, _ptr(filt), _ptr(bias), _ptr(uo), _ptr(x), label, _ptr(after), _ptr(cleared),
                                     out, cap, out_len)
    if not prove:
        hcheck(call(None, 0, None))
        return after, cleared, None
    return after, cleared, flat_out(cap, call)
