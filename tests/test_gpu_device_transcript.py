"""The resident sumcheck tail with its Fiat-Shamir transcript on the device (dp_sc_run_tail_fs, csrc/sumcheck.cu k_sc_res with
sc_res_fs_round; the sponge is csrc/poseidon2.cuh P2Sponge).  In blocking wait mode prove_parallel hands the Poseidon2 duplex state to
the kernel when the resident tail starts and takes it back with every message and challenge; the proof must not change."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O
import test_gpu_sumcheck_dispatch as D

P = O.P
LABEL = b"m2vec"
FS_PROFILE = "k_sc_res(resident cluster rounds with the device transcript)"
HOST_PROFILE_PREFIX = "k_sc_res(resident cluster rounds; "
ROUND_LABEL = [int.from_bytes(b"Internal", "little"), int.from_bytes(b" round", "little")]


class PySponge:
    """DuplexChallenger<F, Poseidon2, 8, 4> (host/transcript.hpp Sponge) over the oracle's permutation, state as dp_sc_run_tail_fs
    exchanges it: [state[0..7], input[0..3], n_input, n_output]"""

    def __init__(self, w):
        w = [int(x) for x in w]
        self.st, self.inp, self.nin, self.nout = w[:8], w[8:12], w[12], w[13]

    def words(self):
        return self.st + self.inp + [self.nin, self.nout]

    def duplex(self):
        for i in range(self.nin):
            self.st[i] = self.inp[i]
        self.nin = 0
        self.st = [int(x) for x in O.poseidon2_permute(np.array(self.st, dtype=np.uint64))]
        self.nout = 4

    def observe(self, v):
        self.nout = 0
        self.inp[self.nin] = int(v)
        self.nin += 1
        if self.nin == 4:
            self.duplex()

    def sample(self):
        if self.nin or not self.nout:
            self.duplex()
        self.nout -= 1
        return self.st[self.nout]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _fs_launches(gpu):
    fs = host = 0
    for name, (count, _, _) in gpu.profile_read().items():
        if name.startswith(FS_PROFILE):
            fs += count
        elif name.startswith(HOST_PROFILE_PREFIX):
            host += count
    return fs, host


def _run_tail(gpu, sc, nv, max_deg, sponge, prev=None):
    """dp_sc_run_tail_fs for the remaining nv rounds: (msgs[nv, max_deg+1, 2], challenges[nv, 2], sponge_out[14])"""
    s_in = np.ascontiguousarray(np.array(sponge, dtype=np.uint64))
    msgs = np.zeros((nv, max_deg + 1, 2), dtype=np.uint64)
    ch = np.zeros((nv, 2), dtype=np.uint64)
    s_out = np.zeros(14, dtype=np.uint64)
    c = None if prev is None else _p(np.ascontiguousarray(np.array(prev, dtype=np.uint64)))
    gpu.check(gpu.lib().dp_sc_run_tail_fs(sc.h, c, _p(s_in), _p(msgs), _p(ch), _p(s_out)))
    return msgs, ch, s_out


SPONGE_STATES = [
    ("fresh", [0] * 8 + [0] * 4 + [0, 0]),
    ("nin1_nout0_zeros", [0] * 8 + [0, 0, 0, 0] + [1, 0]),
    ("nin2_nout0_pminus1", [P - 1] * 8 + [P - 1] * 4 + [2, 0]),
    ("nin3_nout0_mixed", [0, P - 1] * 4 + [P - 1, 0, P - 1, 0] + [3, 0]),
    ("nin0_nout1", list(range(1, 9)) + [9, 10, 11, 12] + [0, 1]),
    ("nin0_nout3_pminus1", [P - 1] * 8 + [0] * 4 + [0, 3]),
    ("nin0_nout4", [int(x) for x in O.splitmix_f(99, 8)] + [0] * 4 + [0, 4]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("max_deg", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("state", [s[0] for s in SPONGE_STATES])
def test_device_sponge_continues_a_handed_over_state(gpu, state, max_deg):
    """Each round absorbs 2 (max_deg + 1) + 2 words (6..14) from a state handed over mid-block (pending inputs, unread outputs,
    words 0 and p - 1): the challenges and the state coming back equal the duplex sponge run over the same words, and the
    messages equal the oracle's at those challenges (points above the product degree extrapolated)."""
    w = dict(SPONGE_STATES)[state]
    nv = 4
    mles = [(O.splitmix_e(5, 1 << nv), True), (O.splitmix_f(6, 1 << nv), False)][:2 if max_deg >= 2 else 1]
    products = [((3, 4), list(range(len(mles))))]
    sc = gpu.Sumcheck([gpu.Mle.upload(a, e) for a, e in mles], products, nv, max_deg)
    try:
        gpu.check(gpu.lib().dp_sc_set_resident_tail(sc.h, 1))
        msgs, ch, s_out = _run_tail(gpu, sc, nv, max_deg, w)
        fin = sc.finish(ch[-1])
    finally:
        sc.destroy()
    ref = PySponge(w)
    for k in range(nv):
        for e in msgs[k]:
            ref.observe(e[0])
            ref.observe(e[1])
        for x in ROUND_LABEL:
            ref.observe(x)
        c0 = ref.sample()
        c1 = ref.sample()
        assert [int(ch[k][0]), int(ch[k][1])] == [c0, c1], "round %d challenge" % k
    assert [int(x) for x in s_out] == ref.words(), "sponge state after the tail"
    exp_msgs, exp_fin = O.sumcheck_rounds_fixed(mles, products, nv, ch)
    d = len(products[0][1])
    for k in range(nv):
        assert (msgs[k][:d + 1] == exp_msgs[k]).all(), "round %d message" % k
        for x in range(d + 1, max_deg + 1):
            assert [int(v) for v in msgs[k][x]] == D._extrapolate(exp_msgs[k], x), "round %d point %d" % (k, x)
    assert (fin == exp_fin).all()


RESIDENT_CASES = [c.name for c in D.CASES if any(r["family"] == "resident" for r in D.dispatch(c.mles, c.products, c.nv, True))]


def _prove(gpu, mles, products, nv):
    """prove_parallel through the host library with an explicit transcript; returns the proof and one challenge drawn after it"""
    prods = gpu.make_products(products)
    max_deg = max(len(p[1]) for p in products)
    point = np.zeros((nv, 2), dtype=np.uint64)
    msgs = np.zeros((nv, max_deg + 1, 2), dtype=np.uint64)
    fin = np.zeros((len(mles), 2), dtype=np.uint64)
    deg = C.c_uint32()
    t = gpu.Transcript(LABEL)
    try:
        gpu.hcheck(gpu.host().dph_sumcheck_prove_parallel(gpu.handles(mles), len(mles), prods, len(products), nv, LABEL, t.h, _p(point), _p(msgs),
                                                          _p(fin), C.byref(deg)))
        after = t.challenge(b"after")
    finally:
        t.free()
    return point, msgs, fin, after


@pytest.mark.gpu
@pytest.mark.parametrize("name", RESIDENT_CASES)
def test_resident_cases_prove_with_the_device_transcript(gpu, name):
    """every resident route of the dispatch matrix (DSEL 0-5, from round 0 and mid-proof, 1-4 CTAs, 48 products / 96 MLEs), proved in
    blocking wait mode: one device-transcript tail, the oracle's proof word for word, and the transcript continues exactly as after
    the host-driven proof in spin mode"""
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
            runs[mode] = _prove(gpu, dm, products, case.nv) + _fs_launches(gpu)
        finally:
            gpu.profile_enable(False)
            gpu.profile_reset()
            gpu.set_wait_mode(before)
    for mode, (point, msgs, fin, after, fs, host) in runs.items():
        what = "%s mode=%d" % (name, mode)
        assert (point == opoint).all() and (msgs == omsgs).all() and (fin == ofin).all(), what
        assert (fs, host) == ((1, 0) if mode == 1 else (0, 1)), what + ": resident launches (device transcript, host transcript)"
    assert (runs[1][3] == runs[0][3]).all(), "%s: transcript state after the proof differs between the two paths" % name


@pytest.mark.gpu
def test_selection_and_refusals(gpu):
    """dp_sc_tail_fs_next says yes only in blocking wait mode and only when the next round starts the resident tail;
    dp_sc_run_tail_fs refuses a round the tail does not serve and a sponge state out of range, then proves the rest mid-proof"""
    nv = 13
    mles = [(O.splitmix_f(s, 1 << nv), False) for s in (1, 2, 3)]
    products = [((1, 0), [0, 1, 2])]
    sc = gpu.Sumcheck([gpu.Mle.upload(a, e) for a, e in mles], products, nv, 3)
    yes = C.c_int(-1)
    before = gpu.lib().dp_get_wait_mode()
    try:
        gpu.check(gpu.lib().dp_sc_set_resident_tail(sc.h, 1))
        gpu.set_wait_mode(1)
        gpu.check(gpu.lib().dp_sc_tail_fs_next(sc.h, C.byref(yes)))
        assert yes.value == 0                                       # 4096 pairs in round 0: not resident yet
        with pytest.raises(gpu.DpError) as e:
            _run_tail(gpu, sc, nv, 3, [0] * 14)
        assert e.value.code == gpu.DP_ERR_STATE
        m0 = sc.round(None)
        ch0 = O.splitmix_e(4, 1)[0]
        gpu.check(gpu.lib().dp_sc_tail_fs_next(sc.h, C.byref(yes)))
        assert yes.value == 1                                       # round 1: 2048 pairs, resident
        gpu.set_wait_mode(0)
        gpu.check(gpu.lib().dp_sc_tail_fs_next(sc.h, C.byref(yes)))
        assert yes.value == 0                                       # spin mode keeps the host transcript
        gpu.set_wait_mode(1)
        bad = [0] * 12 + [4, 0]
        with pytest.raises(gpu.DpError) as e:
            _run_tail(gpu, sc, nv - 1, 3, bad, prev=ch0)
        assert e.value.code == gpu.DP_ERR_INVALID
        msgs, ch, _ = _run_tail(gpu, sc, nv - 1, 3, [0] * 14, prev=ch0)
        fin = sc.finish(ch[-1])
    finally:
        gpu.set_wait_mode(before)
        sc.destroy()
    exp_msgs, exp_fin = O.sumcheck_rounds_fixed(mles, products, nv, np.vstack([ch0[None, :], ch]))
    assert (m0 == exp_msgs[0]).all() and (msgs == exp_msgs[1:]).all() and (fin == exp_fin).all()
