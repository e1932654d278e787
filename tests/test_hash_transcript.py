"""CPU tests: Poseidon2 permutation / duplex challenger / BasicTranscript.  The oracle and the product's
host transcript are independent restatements; they must agree, and both must reproduce the regression
vectors emitted by oracle/gen_poseidon2_constants.py (provenance and what is / is not pinned: see that
script's docstring -- hash parity against the reference is PARTIALLY PINNED)."""
import ctypes as C
import importlib.util
import os
import numpy as np
import oracle_py as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gen():
    spec = importlib.util.spec_from_file_location("gen_p2", os.path.join(ROOT, "oracle", "gen_poseidon2_constants.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_constants_header_is_current():
    import io, contextlib
    g = _gen()
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        g.main()
    assert buf.getvalue() == open(os.path.join(ROOT, "include", "dp_poseidon2_constants.h")).read()


def test_permutation_matches_python_restatement():
    g = _gen()
    rc = g.grain_constants(1, 0, 64, 8, 8, 22, g.P)
    # cross-check vector (recalled upstream KAT, HL 4x4 matrix) -- asserted inside the generator too
    assert g.permute([0] * 8, rc, g.M4_HL) == g.KAT_HL_ZEROS
    for inp in ([0] * 8, list(range(8)), [int(v) for v in O.splitmix_f(9, 8)]):
        assert [int(v) for v in O.poseidon2_permute(inp)] == g.permute(inp, rc, g.M4_P3)


def test_host_permutation_equals_oracle():
    import dpb200
    h = dpb200.host()
    for seed in range(20):
        s = O.splitmix_f(seed, 8)
        mine = s.copy()
        h.dph_poseidon2_permute(mine.ctypes.data_as(C.c_void_p))
        assert (mine == O.poseidon2_permute(s)).all()


def test_compress_is_two_permutations_popped_from_the_end():
    """poseidon/src/poseidon_hash.rs:66-71 over DuplexChallenger<_,_,8,4>: absorb x, permute, absorb y
    (overwrite mode), permute, squeeze state[3],state[2],state[1],state[0]."""
    x, y = O.splitmix_f(1, 4), O.splitmix_f(2, 4)
    st = np.zeros(8, dtype=np.uint64)
    st[:4] = x
    st = O.poseidon2_permute(st)
    st[:4] = y
    st = O.poseidon2_permute(st)
    assert (O.compress(x, y) == st[:4][::-1]).all()


def test_hash_or_noop():
    """<= 4 elements: zero-padded copy, no permutation (poseidon_hash.rs:22-28, digest.rs:24-33)"""
    assert (O.hash_or_noop([5, 6]) == np.array([5, 6, 0, 0], dtype=np.uint64)).all()
    v = O.splitmix_f(3, 6)
    st = np.zeros(8, dtype=np.uint64)
    st[:4] = v[:4]
    st = O.poseidon2_permute(st)
    st[:2] = v[4:]
    st = O.poseidon2_permute(st)
    assert (O.hash_or_noop(v) == st[:4][::-1]).all()


def test_host_transcript_equals_oracle_transcript():
    import dpb200
    to = O.Transcript(b"m2vec")
    th = dpb200.Transcript(b"m2vec")
    f = O.splitmix_f(5, 11)
    e = O.splitmix_e(6, 3)
    for rnd in range(5):
        for t in (to, th):
            t.append_f(f)
            t.append_e(e)
            t.append_msg(b"some label!")
        c1 = to.challenge(b"Internal round")
        out = th.challenge(b"Internal round")
        assert (c1 == out).all()
        assert int(c1[0]) < O.P and int(c1[1]) < O.P
    th.free()


def test_fast_host_permutation_equals_the_canonical_formulation():
    """the weak-form host permutation (host/transcript.hpp) against the plain canonical one on 300k seeded states incl. edge
    values (0, 1, p-1, 2^32-1, 2^32, 2^63, ...) and a chained sponge-like sequence: identical, canonical outputs"""
    import dpb200 as dp
    assert dp.host().dph_poseidon2_selfcheck(300000, 12345) == 0


def test_fast_checker_permutation_equals_the_plain_restatement():
    """oracle/poseidon.hpp: the speed-oriented permutation used by the CPU baseline against the line-by-line restatement"""
    L = O.lib()
    L.dpo_poseidon2_selfcheck.restype = C.c_uint64
    L.dpo_poseidon2_selfcheck.argtypes = [C.c_uint64, C.c_uint64]
    assert L.dpo_poseidon2_selfcheck(300000, 777) == 0
