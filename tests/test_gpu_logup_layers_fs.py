"""The small layers of a LogUp-GKR batch in one resident launch with the transcript on the device (dp_logup_run_layers_fs,
csrc/sumcheck.cu k_logup_res).  In blocking wait mode logup_batch_prove (host/zkml.hpp) hands the leading layers, their sumchecks,
final evaluations and the logup_batching / logup_alpha / logup_lambda draws to the device; the proof and the transcript state after it
must equal the per-layer host path, which spin mode keeps and which the whole-proof tests check against the oracle."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O

P = O.P
LABEL = b"m2vec"
LAYERS_PROFILE = "k_logup_res(resident LogUp-GKR layers, device transcript)"


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _column(pattern, n, seed):
    if pattern == "zero":
        return np.zeros(n, dtype=np.uint64)
    if pattern == "pm1":
        return np.full(n, P - 1, dtype=np.uint64)
    return np.array(O.splitmix_f(seed, n), dtype=np.uint64)


def _prove(gpu, cols, mult, cpi, mode):
    """logup_batch_prove in wait mode `mode`; returns the proof words and the k_logup_res launches"""
    H = gpu.host()
    dm = [gpu.Mle.upload(c, False) for c in cols]
    dmult = gpu.Mle.upload(mult, False) if mult is not None else None
    cc = np.array(O.splitmix_f(91, 2), dtype=np.uint64)
    sc = np.array(O.splitmix_f(92, 2), dtype=np.uint64)
    out = np.zeros(1 << 20, dtype=np.uint64)
    n = C.c_uint64()
    before = gpu.lib().dp_get_wait_mode()
    gpu.set_wait_mode(mode)
    gpu.profile_enable(True)
    gpu.profile_reset()
    try:
        gpu.hcheck(H.dph_logup_prove(gpu.handles(dm), len(dm), dmult.h if dmult else None, cpi, _p(cc), _p(sc), LABEL, _p(out), out.size, C.byref(n)))
        gpu.lib().dp_profile_flush()
        fs = gpu.profile_read().get(LAYERS_PROFILE, (0,))[0]
    finally:
        gpu.profile_enable(False)
        gpu.profile_reset()
        gpu.set_wait_mode(before)
    return out[:n.value].copy(), fs


def _case(kind, n_circuits, cpi, nv, pattern="rand"):
    n = 1 << nv
    if kind == "table":
        cols = [_column(pattern, n, 10 + k) for k in range(2)]
        return cols, _column(pattern if pattern != "rand" else "rand", n, 30), 1
    cols = [_column(pattern, n, 100 + k) for k in range(n_circuits * cpi)]
    return cols, None, cpi


# (kind, circuits, columns_per_instance, log2 column length, pattern): lookup batches of 1, 2, 5 and 7 circuits; 1 or 2 columns per
# instance; nv = 4 puts every layer, the two-view first layer and the lookup's final-round claim on the device; nv = 10 (the flagship's
# 1024-entry columns) and 13 stop the device range before the batch's last layer, so the per-layer path continues from its state
CASES = [
    ("lookup", 1, 1, 4, "rand"), ("lookup", 1, 1, 10, "rand"), ("lookup", 2, 2, 10, "rand"), ("lookup", 5, 1, 10, "rand"),
    ("lookup", 7, 1, 10, "rand"), ("lookup", 5, 2, 4, "rand"), ("lookup", 2, 1, 13, "rand"), ("lookup", 7, 2, 6, "rand"),
    ("lookup", 2, 1, 5, "zero"), ("lookup", 2, 1, 5, "pm1"),
    ("table", 1, 1, 4, "rand"), ("table", 1, 1, 8, "rand"), ("table", 1, 1, 13, "rand"), ("table", 1, 1, 6, "pm1"), ("table", 1, 1, 6, "zero"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=["%s-c%d-cpi%d-nv%d-%s" % c for c in CASES])
def test_device_layers_match_the_host_path(gpu, case):
    kind, nc, cpi, nv, pattern = case
    cols, mult, cpi = _case(kind, nc, cpi, nv, pattern)
    host, fs0 = _prove(gpu, cols, mult, cpi, 0)
    dev, fs1 = _prove(gpu, cols, mult, cpi, 1)
    assert fs0 == 0 and fs1 == 1, "k_logup_res launches: spin %d, blocking %d" % (fs0, fs1)
    assert host.size == dev.size and (host == dev).all(), "proof or transcript state differs from the per-layer host path"


def _circuits(gpu, n_circuits, nv):
    L = gpu.lib()
    cc = np.array([3, 0], dtype=np.uint64)
    sc = np.array([5, 0], dtype=np.uint64)
    keep, hs = [], []
    for k in range(n_circuits):
        m = gpu.Mle.upload(_column("rand", 1 << nv, 200 + k), False)
        h = C.c_void_p()
        gpu.check(L.dp_logup_build((C.c_void_p * 1)(m.h), 1, None, _p(cc), _p(sc), C.byref(h)))
        keep.append(m)
        hs.append(h.value)
    return keep, hs


@pytest.mark.gpu
def test_selection_and_refusals(gpu):
    """the library takes leading layers only in blocking mode, for <= 16 circuits and resident-sized layers; the run entry refuses a
    range it does not take and a sponge state out of range; under BLAKE3 the Poseidon2 k_logup_res count is 0 because the BLAKE3
    instantiation runs instead"""
    L = gpu.lib()
    keep, hs = _circuits(gpu, 17, 10)
    n = C.c_uint32()
    before = L.dp_get_wait_mode()
    try:
        gpu.set_wait_mode(0)
        gpu.check(L.dp_logup_layers_fs_next((C.c_void_p * 1)(hs[0]), 1, 1, C.byref(n)))
        assert n.value == 0                                             # spin mode
        gpu.set_wait_mode(1)
        gpu.check(L.dp_logup_layers_fs_next((C.c_void_p * 1)(hs[0]), 1, 1, C.byref(n)))
        assert n.value == 9                                             # 3 x 2^8 pairs in layer 9: all 9 layers
        gpu.check(L.dp_logup_layers_fs_next((C.c_void_p * 7)(*hs[:7]), 7, 1, C.byref(n)))
        assert n.value == 7                                             # 21 x 2^6 = 1344 <= 2048 < 21 x 2^7
        gpu.check(L.dp_logup_layers_fs_next((C.c_void_p * 7)(*hs[:7]), 7, 8, C.byref(n)))
        assert n.value == 0                                             # an oversize layer
        gpu.check(L.dp_logup_layers_fs_next((C.c_void_p * 17)(*hs), 17, 1, C.byref(n)))
        assert n.value == 0                                             # more circuits than the kernel takes
        z = np.zeros(64, dtype=np.uint64)
        bufs = [np.zeros(1 << 12, dtype=np.uint64) for _ in range(3)]
        args = lambda sp: [_p(z[0:2]), _p(z[2:30]), _p(z[30:32]), _p(z[32:34]), _p(sp)] + [_p(b) for b in bufs]
        with pytest.raises(gpu.DpError) as e:
            gpu.check(L.dp_logup_run_layers_fs((C.c_void_p * 7)(*hs[:7]), 7, 1, 8, *args(np.zeros(14, dtype=np.uint64))))
        assert e.value.code == gpu.DP_ERR_STATE
        bad = np.array([0] * 12 + [4, 0], dtype=np.uint64)
        with pytest.raises(gpu.DpError) as e:
            gpu.check(L.dp_logup_run_layers_fs((C.c_void_p * 1)(hs[0]), 1, 1, 2, *args(bad)))
        assert e.value.code == gpu.DP_ERR_INVALID
    finally:
        gpu.set_wait_mode(before)
        for h in hs:
            L.dp_logup_free(C.c_void_p(h))
    cols, mult, cpi = _case("lookup", 2, 1, 6)
    gpu.set_hasher(1)
    try:
        blake, fs = _prove(gpu, cols, mult, cpi, 1)
        blake0, _ = _prove(gpu, cols, mult, cpi, 0)
    finally:
        gpu.set_hasher(0)
    assert fs == 0 and (blake == blake0).all()
