"""GPU parity tests (-m gpu): Basefold commit / open / batch_open through the C ABI + host mirror against
the oracle -- bit-exact roots, codewords, round messages, final message and every query opening."""
import ctypes as C

import numpy as np
import pytest

import dpb200
import oracle_py as O
from test_oracle_basefold import parse_flat

pytestmark = pytest.mark.gpu


def rnd_poly(seed, nv, ext):
    return O.splitmix_e(seed, 1 << nv) if ext else O.splitmix_f(seed, 1 << nv)


@pytest.mark.parametrize("nv,full_log,ext", [(1, 8, False), (3, 8, True), (7, 10, False), (8, 8, False), (9, 12, False), (10, 10, True),
                                             (12, 14, False), (13, 13, True), (16, 16, False), (18, 20, False)])
def test_commit(gpu, nv, full_log, ext):
    """root, bit-reversed codeword and bit-reversed evaluations (basefold.rs:86-154,304-354)"""
    ev = rnd_poly(100 + nv, nv, ext)
    root, cw, bh = O.pcs_commit(ev, ext, full_log)
    c = gpu.Commitment(gpu.Mle.upload(ev, ext), full_log)
    assert c.num_vars == nv and c.is_base == (not ext) and c.trivial == (nv <= 7)
    assert (c.bh_evals() == bh).all()
    assert (c.codeword() == cw).all()
    assert (c.root == root).all()


def test_commit_too_large(gpu):
    with pytest.raises(gpu.DpError) as e:
        gpu.Commitment(gpu.Mle.upload(O.splitmix_f(1, 1 << 9), False), 8)
    assert "PolynomialTooLarge" in str(e.value)


@pytest.mark.parametrize("nv,full_log,ext", [(8, 8, False), (9, 11, False), (10, 10, True), (12, 12, False), (14, 16, False), (15, 15, True)])
def test_open(gpu, nv, full_log, ext):
    """whole opening proof (commit_phase.rs:30-183 + query_phase.rs:31-65,373-417), same transcript"""
    ev = rnd_poly(200 + nv, nv, ext)
    pt = O.splitmix_e(300 + nv, nv)
    exp = O.pcs_open(ev, ext, full_log, pt)
    root, got = gpu.pcs_open(gpu.Mle.upload(ev, ext), full_log, pt)
    assert (root == O.pcs_commit(ev, ext, full_log, want_codeword=False)[0]).all()
    assert got.shape == exp.shape
    if not (got == exp).all():
        a, b = parse_flat(got), parse_flat(exp)
        for k in ("sumcheck_messages", "roots", "final_message"):
            assert a[k] == b[k], k
        assert a["single"] == b["single"], "queries"
    assert (got == exp).all()
    assert O.pcs_verify(got, root, nv, not ext, full_log, pt, O.evaluate(ev, ext, pt)) is None   # Basefold::verify accepts (basefold.rs:863-962)


@pytest.mark.parametrize("shape,full_log", [([(10, False)], 10), ([(10, False), (8, False), (9, True)], 10), ([(9, False), (12, False), (12, True), (8, False)], 13),
                                            ([(14, False), (14, False), (11, False)], 14)])
def test_batch_open(gpu, shape, full_log):
    """batch_open (basefold.rs:546-770): classic sumcheck + batch_commit_phase + batched queries"""
    polys = [(rnd_poly(400 + 7 * i + nv, nv, ext), ext) for i, (nv, ext) in enumerate(shape)]
    pts = [O.splitmix_e(500 + i, nv) for i, (nv, _) in enumerate(shape)]
    exp = O.pcs_batch_open(polys, full_log, pts)
    got = gpu.pcs_batch_open([gpu.Mle.upload(a, e) for a, e in polys], full_log, pts)
    assert got.shape == exp.shape
    if not (got == exp).all():
        a, b = parse_flat(got), parse_flat(exp)
        for k in ("sumcheck_proof", "sumcheck_messages", "roots", "final_message"):
            assert a[k] == b[k], k
        assert a["batched"] == b["batched"], "queries"
    assert (got == exp).all()
    # the device's proof is accepted by the restated Basefold::batch_verify (basefold.rs:964-1098)
    roots = np.array([O.pcs_commit(p, e, full_log, want_codeword=False)[0] for p, e in polys])
    evals = np.array([O.evaluate(p, e, pt) for (p, e), pt in zip(polys, pts)])
    assert O.pcs_batch_verify(got, roots, [nv for nv, _ in shape], [not e for _, e in shape], full_log, pts, evals) is None


def test_open_full_size_properties(gpu):
    """BASELINE cfg-4 scale-down (nu=20; 2^24 is exercised by bench.py): properties that do not need the
    oracle at full size -- the commit-phase sumcheck chains (2 c0 + c1 + c2 == previous claim evaluated at
    the challenge is checked by re-deriving the claim from the final message), and every opened pair
    authenticates against its root."""
    from test_oracle_basefold import authenticate
    nv, full_log = 20, 20
    ev = O.splitmix_f(9, 1 << nv)
    pt = O.splitmix_e(10, nv)
    m = gpu.Mle.upload(ev, False)
    root, flat = gpu.pcs_open(m, full_log, pt)
    pr = parse_flat(flat)
    assert len(pr["sumcheck_messages"]) == nv - 7 and len(pr["roots"]) == nv - 8 and len(pr["single"]) == 200
    assert O.pcs_verify(flat, root, nv, True, full_log, pt, O.evaluate(ev, False, pt)) is None   # the verifier needs no 2^20-sized work
    m0 = pr["sumcheck_messages"][0]
    s = O.pe_add(O.pe_add(O.pe_add((m0[0], m0[1]), (m0[0], m0[1])), (m0[2], m0[3])), (m0[4], m0[5]))
    assert s == tuple(int(x) for x in m.evaluate(pt))
    for qr in pr["single"][:25]:
        assert authenticate(qr["commitment"], [int(x) for x in root], True)
        for k, oq in enumerate(qr["oracle"]):
            assert authenticate(oq, pr["roots"][k], False)


@pytest.mark.parametrize("n_polys,nv,full_log,ext", [(3, 9, 10, False), (5, 10, 10, False), (2, 9, 9, True), (1, 9, 9, False), (4, 8, 12, False), (6, 13, 13, False), (3, 16, 16, False), (3, 5, 8, False)])
def test_batch_commit_and_simple_batch_open(gpu, n_polys, nv, full_log, ext):
    """Basefold::batch_commit (one tree with batch leaves) and simple_batch_open (basefold.rs:356-452,777-861): root and whole
    proof identical to the CPU checker's, and accepted by the restated simple_batch_verify"""
    polys = [rnd_poly(900 + i, nv, ext) for i in range(n_polys)]
    pt = O.splitmix_e(950, nv)
    if nv <= 7:   # trivial commitment: only the root (the opening is the evaluations themselves)
        root, _ = gpu.pcs_simple_batch([gpu.Mle.upload(p, ext) for p in polys], full_log)
        assert (root == O.pcs_simple_batch(polys, ext, full_log)[0]).all()
        return
    eroot, evals, exp = O.pcs_simple_batch(polys, ext, full_log, pt)
    root, got = gpu.pcs_simple_batch([gpu.Mle.upload(p, ext) for p in polys], full_log, pt, evals)
    assert (root == eroot).all()
    assert got.shape == exp.shape and (got == exp).all()
    assert O.pcs_simple_batch_verify(got, root, nv, not ext, n_polys, full_log, pt, evals) is None


def test_batch_open_with_shared_points(gpu):
    """batch_open where two polynomials share a point and one polynomial is opened at two points (the merged-polynomial case of
    basefold.rs:617-640): the device adds one sumcheck product per evaluation instead of merging; identical proof"""
    shape = [(10, False), (10, False), (9, True), (10, False)]
    polys = [(rnd_poly(1000 + i, nv, ext), ext) for i, (nv, ext) in enumerate(shape)]
    points = [O.splitmix_e(1100, 10), O.splitmix_e(1101, 9), O.splitmix_e(1102, 10)]
    eval_poly, eval_point = [0, 1, 2, 3, 0], [0, 0, 1, 2, 2]
    exp, _, _ = O.pcs_batch_open_evals(polys, 11, points, eval_poly, eval_point)
    got = gpu.pcs_batch_open_evals([gpu.Mle.upload(a, e) for a, e in polys], 11, points, eval_poly, eval_point)
    assert got.shape == exp.shape and (got == exp).all()


# ---- refusals of the Basefold C ABI ------------------------------------------------------------------------------------------------
def _commit(gpu, nv, full_log):
    return gpu.Commitment(gpu.Mle.upload(rnd_poly(600 + nv, nv, False), False), full_log)


def _open_begin(gpu, handles, num_vars, batch=False):
    """dp_pcs_open_begin over raw commitment handles -> return code (an opening that starts is freed again)"""
    L = gpu.lib()
    hs = (C.c_void_p * len(handles))(*handles)
    pt = gpu._u64(O.splitmix_e(610, num_vars)).reshape(-1)
    coeffs = np.ones(2 * len(handles), dtype=np.uint64) if batch else None
    o, msg = C.c_void_p(), np.zeros(6, dtype=np.uint64)
    rc = L.dp_pcs_open_begin(hs, None if coeffs is None else coeffs.ctypes.data, len(handles), pt.ctypes.data, num_vars, C.byref(o), msg.ctypes.data)
    if rc == 0:
        L.dp_pcs_open_free(o)
    return rc


def _open_trivial(gpu):
    c = _commit(gpu, 5, 8)
    return _open_begin(gpu, [c.h.value], 5)


def _open_larger(gpu):
    c = _commit(gpu, 10, 10)
    return _open_begin(gpu, [c.h.value], 9)


def _open_few_vars(gpu):
    # every non-trivial commitment has more than 7 variables, so the size check above comes first and its message wins
    c = _commit(gpu, 8, 8)
    return _open_begin(gpu, [c.h.value], 7)


def _open_single_wrong_vars(gpu):
    c = _commit(gpu, 9, 10)
    return _open_begin(gpu, [c.h.value], 10)


def _sharded(gpu, nv=13):
    L = gpu.lib()
    m, h = gpu.Mle.upload(rnd_poly(620, nv, False), False), C.c_void_p()
    gpu.check(L.dp_pcs_commit_shard(m.h, nv, 0, 2, C.byref(h)))
    return h


def _open_sharded_in_batch(gpu):
    h = _sharded(gpu)
    try:
        return _open_begin(gpu, [h.value], 13, batch=True)
    finally:
        gpu.lib().dp_pcs_comm_free(h)


def _open_sharded_without_roots(gpu):
    h = _sharded(gpu)
    try:
        return _open_begin(gpu, [h.value], 13)
    finally:
        gpu.lib().dp_pcs_comm_free(h)


def _shard(gpu, nv, rank, world, hasher=0):
    L = gpu.lib()
    m, h = gpu.Mle.upload(rnd_poly(630, nv, False), False), C.c_void_p()
    gpu.set_hasher(hasher)
    try:
        rc = L.dp_pcs_commit_shard(m.h, nv, rank, world, C.byref(h))
    finally:
        gpu.set_hasher(0)
    if rc == 0:
        L.dp_pcs_comm_free(h)
    return rc


def _batch(gpu, nvs):
    L = gpu.lib()
    mles = [gpu.Mle.upload(rnd_poly(640 + i, nv, False), False) for i, nv in enumerate(nvs)]
    h = C.c_void_p()
    rc = L.dp_pcs_batch_commit(gpu.handles(mles), len(mles), 10, C.byref(h))
    if rc == 0:
        L.dp_pcs_comm_free(h)
    return rc


E = dpb200
REFUSALS = {   # case -> (call, return code, dp_last_error text)
    "open trivial commitment": (_open_trivial, E.DP_ERR_INVALID, "dp_pcs_open_begin: trivial commitment (open it on the host)"),
    "open commitment larger than the opening": (_open_larger, E.DP_ERR_INVALID, "dp_pcs_open_begin: commitment larger than the opening"),
    "open num_vars <= 7": (_open_few_vars, E.DP_ERR_INVALID, "dp_pcs_open_begin: commitment larger than the opening"),
    "single open with the wrong num_vars": (_open_single_wrong_vars, E.DP_ERR_INVALID,
                                            "dp_pcs_open_begin: single open needs one commitment of num_vars variables"),
    "sharded commitment in a batch": (_open_sharded_in_batch, E.DP_ERR_UNSUPPORTED, "dp_pcs_open_begin: a sharded commitment is opened alone"),
    "sharded commitment without its shard roots": (_open_sharded_without_roots, E.DP_ERR_STATE,
                                                   "dp_pcs_open_begin: sharded commitment needs num_vars variables and its shard roots set"),
    "shard over a world that is not a power of two": (lambda g: _shard(g, 13, 0, 3), E.DP_ERR_INVALID,
                                                      "dp_pcs_commit_shard: world must be a power of two >= 2 and rank < world"),
    "shard with rank >= world": (lambda g: _shard(g, 13, 2, 2), E.DP_ERR_INVALID,
                                 "dp_pcs_commit_shard: world must be a power of two >= 2 and rank < world"),
    "shard a polynomial that is too small": (lambda g: _shard(g, 12, 0, 2), E.DP_ERR_INVALID,
                                             "dp_pcs_commit_shard: polynomial too small to shard over this many ranks"),
    "shard under BLAKE3": (lambda g: _shard(g, 13, 0, 2, hasher=1), E.DP_ERR_UNSUPPORTED, "dp_pcs_commit_shard: Poseidon2 trees only"),
    "batch commit of 0 polynomials": (lambda g: _batch(g, []), E.DP_ERR_INVALID, "cannot batch commit to zero polynomials"),
    "batch commit of 65 polynomials": (lambda g: _batch(g, [8] * 65), E.DP_ERR_UNSUPPORTED, "dp_pcs_batch_commit: at most 64 polynomials per batch"),
    "batch commit of mixed sizes": (lambda g: _batch(g, [9, 10]), E.DP_ERR_INVALID,
                                    "cannot batch commit to polynomials with different number of variables"),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_abi_refusal(gpu, case):
    """each refusal returns its code and message, and the context it happened in still commits and opens like the oracle"""
    call, code, text = REFUSALS[case]
    assert call(gpu) == code
    assert gpu.lib().dp_last_error().decode() == text
    ev, pt = rnd_poly(650, 9, False), O.splitmix_e(651, 9)
    root, got = gpu.pcs_open(gpu.Mle.upload(ev, False), 10, pt)
    assert (root == O.pcs_commit(ev, False, 10, want_codeword=False)[0]).all()
    assert (got == O.pcs_open(ev, False, 10, pt)).all()
