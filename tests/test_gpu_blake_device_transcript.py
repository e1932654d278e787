"""BlakeTranscript on the device (dp_sc_run_tail_fs_blake, dp_logup_run_layers_fs_blake; csrc/blake3.cuh TrB3 over the incremental
BLAKE3 there).  Under the `blake` hasher a prover in blocking wait mode hands its transcript's hasher image to the resident
sumcheck tail and to the LogUp-GKR layer kernel and takes it back with every message and challenge.  Everything here is pinned: the
challenges against the Python `blake3` package, the proofs against the checker's BLAKE3 proofs."""
import ctypes as C
import json
import os

import numpy as np
import pytest

blake3 = pytest.importorskip("blake3")
import models  # noqa: E402
import oracle_py as O  # noqa: E402
import test_blake as TB  # noqa: E402
import test_blake_transcript_state as TS  # noqa: E402
import test_gpu_device_transcript as DT  # noqa: E402
import test_gpu_logup_layers_fs as LG  # noqa: E402
import test_gpu_sumcheck_dispatch as D  # noqa: E402

pytestmark = pytest.mark.gpu
P = O.P
WORDS = 80
LABEL = b"m2vec"
B3_TAIL = "k_sc_res(resident cluster rounds, BLAKE3 device transcript)"
B3_LAYERS = "k_logup_res(resident LogUp-GKR layers, BLAKE3 transcript)"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "blake_retry.json")
PREFIXES = [0, 1, 63, 64, 65, 1023, 1024, 1025, 2047, 2048, 3072, 4096, 8192, 20480]


@pytest.fixture()
def blake(gpu):
    O.set_hash_mode(1); gpu.set_hasher(1)
    yield gpu
    O.set_hash_mode(0); gpu.set_hasher(0)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _host_t(gpu, label=b"", image=None):
    """a host BlakeTranscript (the `blake` hasher must be selected), continued from `image` when given"""
    t = gpu.Transcript(label)
    if image is not None:
        t.load_state(2, image)
    return t


def _image(t):
    kind, w = t.save_state()
    assert kind == 2
    return w


def _run_tail(gpu, sc, nv, max_deg, image, prev=None, entry="dp_sc_run_tail_fs_blake"):
    """the remaining nv rounds on the device: (msgs[nv, max_deg+1, 2], challenges[nv, 2], image_out[80])"""
    w_in = np.ascontiguousarray(np.array(image, dtype=np.uint64))
    msgs = np.zeros((nv, max_deg + 1, 2), dtype=np.uint64)
    ch = np.zeros((nv, 2), dtype=np.uint64)
    w_out = np.zeros(WORDS, dtype=np.uint64)
    c = None if prev is None else _p(np.ascontiguousarray(np.array(prev, dtype=np.uint64)))
    gpu.check(getattr(gpu.lib(), entry)(sc.h, c, _p(w_in), _p(msgs), _p(ch), _p(w_out)))
    return msgs, ch, w_out


def _tail_case(gpu, image, max_deg, nv=4, mles=None, products=None):
    """a sumcheck from round 0 on the device from `image`: messages, challenges, image after; checks the messages against the oracle"""
    mles = mles or [(O.splitmix_e(5, 1 << nv), True), (O.splitmix_f(6, 1 << nv), False)][:2 if max_deg >= 2 else 1]
    products = products or [((3, 4), list(range(len(mles))))]
    sc = gpu.Sumcheck([gpu.Mle.upload(a, e) for a, e in mles], products, nv, max_deg)
    try:
        gpu.check(gpu.lib().dp_sc_set_resident_tail(sc.h, 1))
        msgs, ch, w_out = _run_tail(gpu, sc, nv, max_deg, image)
        fin = sc.finish(ch[-1])
    finally:
        sc.destroy()
    exp_msgs, exp_fin = O.sumcheck_rounds_fixed(mles, products, nv, ch)
    d = len(products[0][1])
    for k in range(nv):
        assert (msgs[k][:d + 1] == exp_msgs[k]).all(), "round %d message" % k
        for x in range(d + 1, max_deg + 1):
            assert [int(v) for v in msgs[k][x]] == D._extrapolate(exp_msgs[k], x), "round %d point %d" % (k, x)
    assert (fin == exp_fin).all()
    return msgs, ch, w_out


def _continue(t, msgs):
    """what the host transcript t draws for these round messages"""
    out = []
    for m in msgs:
        t.append_e(m)
        out.append(tuple(int(x) for x in t.challenge(b"Internal round")))
    return out


# ---- 1. handed-over states -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("max_deg", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("n", PREFIXES)
def test_device_hasher_continues_a_handed_over_state(blake, n, max_deg):
    """the transcript after n label bytes (stack lengths 0 to 3, a pending full block or chunk) continues on the device: the
    challenges equal the package's, the image coming back equals the host hasher's after the same bytes, and the messages equal the
    oracle's at those challenges"""
    label = TS._label(n)
    src = _host_t(blake, label)
    try:
        image = _image(src)
        msgs, ch, w_out = _tail_case(blake, image, max_deg)
        host = _continue(src, msgs)
        host_image = _image(src)
    finally:
        src.free()
    py = TB.PyBlakeTranscript(label)
    for k, m in enumerate(msgs):
        for e in m:
            py.append_e(int(e[0]), int(e[1]))
        assert (int(ch[k][0]), int(ch[k][1])) == py.challenge(b"Internal round") == host[k], "round %d challenge" % k
    assert (w_out == host_image).all(), "image after the tail"


# ---- 2. synthetic images ------------------------------------------------------------------------------------------------------
def _synthetic_high_counter():
    """a valid image with chunk_counter >= 2^32 (the high counter word): three stack entries, 40 bytes in the third block"""
    w = np.zeros(WORDS, dtype=np.uint64)
    w[0:4] = O.splitmix_f(71, 4); w[4] = (1 << 32) | 5; w[13] = 40; w[14] = 2; w[15] = 3
    w[5:10] = O.splitmix_f(72, 5)
    for i in range(3):
        w[16 + 4 * i: 20 + 4 * i] = O.splitmix_f(80 + i, 4)
    return w


@pytest.mark.parametrize("kind", ["stack16", "counter_above_2e32"])
def test_device_hasher_on_synthetic_images(blake, kind):
    if kind == "stack16":
        src = _host_t(blake, TS._label((2 ** 16 - 1) * 1024 + 1))
        image = _image(src)
        assert int(image[15]) == 16
        src.free()
    else:
        image = _synthetic_high_counter()
    t = _host_t(blake, b"", image)
    try:
        assert (_image(t) == image).all()
        msgs, ch, w_out = _tail_case(blake, image, 3, nv=6)
        host = _continue(t, msgs)
        host_image = _image(t)
    finally:
        t.free()
    assert [(int(a), int(b)) for a, b in ch] == host
    assert (w_out == host_image).all()


# ---- 3. the retry path --------------------------------------------------------------------------------------------------------
def test_retry_path(blake):
    """a frozen state (tests/golden/make_blake_retry.py) whose round-0 challenge draws a limb >= p the first time: the device retries
    exactly as read_challenge does"""
    g = json.load(open(GOLDEN))
    label = g["label"].encode()
    mles = [(O.splitmix_e(s, 1 << g["nv"]) if ext else O.splitmix_f(s, 1 << g["nv"]), ext) for s, ext in g["mles"]]
    products = [(tuple(g["product"][0]), g["product"][1])]
    src = _host_t(blake, label)
    try:
        msgs, ch, w_out = _tail_case(blake, _image(src), g["max_deg"], nv=g["nv"], mles=mles, products=products)
        host = _continue(src, msgs)
        host_image = _image(src)
    finally:
        src.free()
    py = TB.PyBlakeTranscript(label)
    for e in msgs[0]:
        py.append_e(int(e[0]), int(e[1]))
    py.append_msg(b"Internal round")
    h = py.h.copy(); h.update(b"challenge")
    o = h.digest(length=16)
    first = [int.from_bytes(o[:8], "little"), int.from_bytes(o[8:], "little")]
    assert first == g["first_attempt"] and max(first) >= P, "the frozen state no longer retries"
    assert (int(ch[0][0]), int(ch[0][1])) == py.read_challenge() == host[0]
    assert [(int(a), int(b)) for a, b in ch] == host
    assert (w_out == host_image).all()


# ---- 4. every resident route through the host library -------------------------------------------------------------------------
def _launches(gpu, name):
    gpu.lib().dp_profile_flush()
    return sum(v[0] for k, v in gpu.profile_read().items() if k == name)


@pytest.mark.parametrize("name", DT.RESIDENT_CASES)
def test_resident_cases_prove_with_the_blake_device_transcript(blake, name):
    """prove_parallel under `blake` in both wait modes: the checker's BLAKE3 proof word for word, one BLAKE3-device-transcript launch
    in blocking mode and none in spin mode, and the transcript continues identically afterwards"""
    gpu = blake
    case = D.CASE_BY_NAME[name]
    mles, products = D.make_inputs(case)
    opoint, omsgs, ofin = O.sumcheck_prove(mles, products, case.nv, LABEL)
    dm = [gpu.Mle.upload(a, e) for a, e in mles]
    runs = {}
    for mode in (0, 1):
        before = gpu.lib().dp_get_wait_mode()
        gpu.set_wait_mode(mode)
        gpu.profile_enable(True)
        gpu.profile_reset()
        try:
            runs[mode] = DT._prove(gpu, dm, products, case.nv) + (_launches(gpu, B3_TAIL), _launches(gpu, DT.FS_PROFILE))
        finally:
            gpu.profile_enable(False)
            gpu.profile_reset()
            gpu.set_wait_mode(before)
    for mode, (point, msgs, fin, after, b3, p2) in runs.items():
        what = "%s mode=%d" % (name, mode)
        assert (point == opoint).all() and (msgs == omsgs).all() and (fin == ofin).all(), what
        assert (b3, p2) == ((1, 0) if mode == 1 else (0, 0)), what + ": BLAKE3 / Poseidon2 device-transcript launches"
    assert (runs[1][3] == runs[0][3]).all(), "%s: transcript state after the proof differs between the two paths" % name


# ---- 5. LogUp-GKR layers ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", LG.CASES, ids=["%s-c%d-cpi%d-nv%d-%s" % c for c in LG.CASES])
def test_blake_device_layers_match_the_host_path(blake, case):
    gpu = blake
    kind, nc, cpi, nv, pattern = case
    cols, mult, cpi = LG._case(kind, nc, cpi, nv, pattern)
    got = {mode: LG._prove(gpu, cols, mult, cpi, mode) for mode in (0, 1)}    # proof words, Poseidon2 k_logup_res launches
    # the BLAKE3 launches, counted on a third blocking run
    before = gpu.lib().dp_get_wait_mode()
    gpu.set_wait_mode(1)
    gpu.profile_enable(True)
    gpu.profile_reset()
    try:
        H = gpu.host()
        dm = [gpu.Mle.upload(c, False) for c in cols]
        dmult = gpu.Mle.upload(mult, False) if mult is not None else None
        cc = np.array(O.splitmix_f(91, 2), dtype=np.uint64)
        sc = np.array(O.splitmix_f(92, 2), dtype=np.uint64)
        out = np.zeros(1 << 20, dtype=np.uint64)
        n = C.c_uint64()
        gpu.hcheck(H.dph_logup_prove(gpu.handles(dm), len(dm), dmult.h if dmult else None, cpi, _p(cc), _p(sc), LABEL, _p(out), out.size, C.byref(n)))
        b3 = _launches(gpu, B3_LAYERS)
    finally:
        gpu.profile_enable(False)
        gpu.profile_reset()
        gpu.set_wait_mode(before)
    (host, p2_0), (dev, p2_1) = got[0], got[1]
    assert p2_0 == 0 and p2_1 == 0, "no Poseidon2 k_logup_res launch under blake"
    assert b3 == 1, "BLAKE3 k_logup_res launches in blocking mode: %d" % b3
    assert host.size == dev.size and (host == dev).all(), "proof or transcript state differs from the per-layer host path"
    assert (out[:n.value] == dev).all()


# ---- 6. refusals --------------------------------------------------------------------------------------------------------------
def test_refusals(blake):
    """each malformed-image rule is DP_ERR_INVALID on both entry points; a round the tail does not serve and a layer range the kernel
    does not take are DP_ERR_STATE"""
    gpu = blake
    L = gpu.lib()
    ok, bad = TS.malformed_images()
    nv = 13
    mles = [(O.splitmix_f(s, 1 << nv), False) for s in (1, 2, 3)]
    sc = gpu.Sumcheck([gpu.Mle.upload(a, e) for a, e in mles], [((1, 0), [0, 1, 2])], nv, 3)
    keep, hs = LG._circuits(gpu, 7, 10)
    before = L.dp_get_wait_mode()
    z = np.zeros(64, dtype=np.uint64)
    bufs = [np.zeros(1 << 12, dtype=np.uint64) for _ in range(3)]
    args = lambda w: [_p(z[0:2]), _p(z[2:30]), _p(z[30:32]), _p(z[32:34]), _p(w)] + [_p(b) for b in bufs]
    try:
        gpu.check(L.dp_sc_set_resident_tail(sc.h, 1))
        gpu.set_wait_mode(1)
        with pytest.raises(gpu.DpError) as e:
            _run_tail(gpu, sc, nv, 3, ok)                                # round 0: 4096 pairs, not resident
        assert e.value.code == gpu.DP_ERR_STATE
        sc.round(None)
        ch0 = O.splitmix_e(4, 1)[0]
        for name, w in bad:
            with pytest.raises(gpu.DpError) as e:
                _run_tail(gpu, sc, nv - 1, 3, w, prev=ch0)
            assert e.value.code == gpu.DP_ERR_INVALID, name
            with pytest.raises(gpu.DpError) as e:
                gpu.check(L.dp_logup_run_layers_fs_blake((C.c_void_p * 1)(hs[0]), 1, 1, 2, *args(w.copy())))
            assert e.value.code == gpu.DP_ERR_INVALID, name
        with pytest.raises(gpu.DpError) as e:
            gpu.check(L.dp_logup_run_layers_fs_blake((C.c_void_p * 7)(*hs[:7]), 7, 1, 8, *args(ok.copy())))
        assert e.value.code == gpu.DP_ERR_STATE                          # layer 8 of 7 circuits is not resident
        msgs, ch, _ = _run_tail(gpu, sc, nv - 1, 3, ok, prev=ch0)       # the handle still proves the rest
        sc.finish(ch[-1])
    finally:
        gpu.set_wait_mode(before)
        sc.destroy()
        for h in hs:
            L.dp_logup_free(C.c_void_p(h))


# ---- 7. whole proofs ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["mlp_2x64", "cnn_small", "token_mlp"])
def test_concurrent_blake_proofs(blake, model):
    """dph_zkml_prove_concurrent_all in blocking wait mode under `blake`: every proof equals the checker's BLAKE3 proof, which the
    restated verifier accepts, and the BLAKE3 device transcript ran"""
    gpu = blake
    if model == "mlp_2x64":
        w, b, rq = O.synthetic_mlp(2, 64, 5)
        x = O.synthetic_input(64, 6)
        ctx = gpu.ZkmlContext(2, 64, w, b, rq)
        exp, _ = O.zkml_prove(2, 64, 5, 6)
        verdict = O.zkml_prove_verify(2, 64, 5, 6)
    else:
        if model == "cnn_small":
            desc, data, x, _ = models.cnn_small(seed=3)
        else:
            desc, data, x = models.token_mlp(seed=11, tokens=8, d_model=32, d_hidden=64)
        ctx = gpu.ModelContext(desc, data, x.size)
        exp, _ = O.model_prove(desc, data, x)
        verdict = O.model_prove_verify(desc, data, x)
    assert verdict is None, verdict
    ctx.run_inference(x)
    before = gpu.lib().dp_get_wait_mode()
    gpu.set_wait_mode(1)
    gpu.profile_enable(True)
    gpu.profile_reset()
    try:
        _, proofs, _ = ctx.prove_concurrent_all(4, 8, stride=exp.size + 64)
        b3 = _launches(gpu, B3_TAIL) + _launches(gpu, B3_LAYERS)
    finally:
        gpu.profile_enable(False)
        gpu.profile_reset()
        gpu.set_wait_mode(before)
        ctx.free()
    for j, got in enumerate(proofs):
        assert got.size == exp.size and (got == exp).all(), "%s: job %d" % (model, j)
    assert b3 > 0, "%s: no BLAKE3 device-transcript launch" % model
