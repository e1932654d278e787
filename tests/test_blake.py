"""The `blake` variant of the path (reference feature flag: mpcs/src/lib.rs:339-342 BlakeHasher, transcript/src/blake.rs BlakeTranscript,
zkml/src/bin/bench.rs:29-44) is fully determined by the reference's sources plus standard BLAKE3 -- no un-vendored constants -- so it
is the variant whose digests, challenges and proof bytes can be PINNED:
  * include/dp_blake3.h  ==  the Python `blake3` package (hash, incremental updates, finalize in the middle, extendable output);
  * the checker's and the host library's BlakeTranscript  ==  a pure-Python restatement of transcript/src/blake.rs on that package;
  * BlakeHasher::{hash_bases, hash_two_digests}  ==  the same;
  * whole proofs under blake: the restated verifiers accept on a fresh BlakeTranscript (CPU), and the device path equals the checker
    word for word (tests/test_gpu_blake.py)."""
import ctypes as C
import numpy as np
import pytest
import oracle_py as O

blake3 = pytest.importorskip("blake3")
P = 0xFFFFFFFF00000001


@pytest.fixture()
def blake_checker():
    O.set_hash_mode(1)
    yield
    O.set_hash_mode(0)


def test_blake3_primitive_matches_the_python_package():
    rng = np.random.default_rng(1)
    L = O.lib()
    for n in [0, 1, 2, 3, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025, 2048, 2049, 3071, 3072, 3073, 4096, 5000, 8192, 8193, 16384, 31744, 65537, 100000]:
        data = rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
        for piece, mid, ol in [(0, 0, 32), (1 if n < 3000 else 977, 0, 32), (64, 0, 64), (1000, n // 2, 100), (1024, 1024 if n > 1024 else 0, 16), (37, 33, 200)]:
            out = (C.c_uint8 * ol)()
            L.dpo_blake3(data, C.c_uint64(n), C.c_uint64(piece), C.c_uint64(mid), out, C.c_uint64(ol))
            assert bytes(out) == blake3.blake3(data).digest(length=ol), (n, piece, mid, ol)


class PyBlakeTranscript:
    """transcript/src/blake.rs through trait Transcript<E> (transcript/src/lib.rs:22-93), on the Python blake3 package"""

    def __init__(self, label):
        self.h = blake3.blake3(); self.h.update(label)

    @staticmethod
    def fe_bytes(v):          # prime_to_bytes: as_canonical_biguint().to_bytes_le()
        v %= P
        return v.to_bytes(8, "little").rstrip(b"\0") or b"\0"

    def append_f(self, v):
        self.h.update(b"field_element"); self.h.update(self.fe_bytes(v))

    def append_msg(self, m):  # trait default: bytes_to_field_elements (8-byte LE chunks, zero padded), then one append each
        for i in range(0, len(m), 8):
            self.append_f(int.from_bytes(m[i:i + 8].ljust(8, b"\0"), "little"))

    def append_e(self, c0, c1):
        self.h.update(b"field_element_ext"); self.h.update(self.fe_bytes(c0) + self.fe_bytes(c1))

    def read_challenge(self):
        while True:
            self.h.update(b"challenge")
            o = self.h.digest(length=16)
            a, b = int.from_bytes(o[:8], "little"), int.from_bytes(o[8:], "little")
            if a < P and b < P:
                return a, b

    def challenge(self, label):
        self.append_msg(label); return self.read_challenge()


def _script(t_new, t_f, t_msg, t_e, t_ch, t_read):
    """the same sequence of transcript operations on any implementation; returns the challenges"""
    out = []
    t = t_new(b"m2vec")
    t_f(t, [0, 1, 255, 256, P - 1, 1 << 32, (1 << 56) + 7])
    t_msg(t, b"Internal round")
    out.append(t_ch(t, b"table_constant"))
    t_e(t, [(0, 0), (1, 0), (0, 1), (P - 1, 123456789012345), (1 << 40, 1 << 48)])
    out.append(t_read(t)); out.append(t_read(t))
    t_msg(t, (20).to_bytes(8, "little")); t_msg(t, bytes(range(1, 33)))           # usize, a 32-byte digest
    t_f(t, [0xFFFFFFFFFFFFFFFF % P, 0xFFFFFFFF00000002 % P])
    for i in range(40):
        t_e(t, [(i * 977 % P, (i + 3) ** 5 % P)]); out.append(t_ch(t, b"Internal round"))
    return out


def host_transcript_ops():
    """_script's operations on dpb200.Transcript, challenges as int pairs; read_challenge is a challenge with an empty label, which
    appends nothing"""
    def ch(t, label):
        return tuple(int(x) for x in t.challenge(label))
    return (lambda t, f: t.append_f(f), lambda t, m: t.append_msg(m), lambda t, e: t.append_e(e), ch, lambda t: ch(t, b""))


def test_checker_and_host_blake_transcripts_match_the_python_restatement(blake_checker):
    py = _script(lambda l: PyBlakeTranscript(l), lambda t, f: [t.append_f(x) for x in f], lambda t, m: t.append_msg(m),
                 lambda t, e: [t.append_e(*x) for x in e], lambda t, l: t.challenge(l), lambda t: t.read_challenge())

    def orc_new(label):
        return O.Transcript(label)
    orc = _script(orc_new, lambda t, f: t.append_f(f), lambda t, m: t.append_msg(m), lambda t, e: t.append_e(e),
                  lambda t, l: tuple(int(x) for x in t.challenge(l)), lambda t: tuple(int(x) for x in t.read_challenge()))
    assert orc == py
    # the product's host library (no GPU needed for the transcript)
    import dpb200 as dp
    # set_hasher also switches the device library's Merkle hasher flag (a plain flag: no device needed)
    dp.set_hasher(1)
    try:
        host = _script(dp.Transcript, *host_transcript_ops())
        assert host == py
    finally:
        dp.set_hasher(0)


def test_blake_hasher_digests(blake_checker):
    L = O.lib()
    rng = np.random.default_rng(3)
    for n in [1, 2, 4, 5, 8, 9, 64, 128, 300]:
        v = (rng.integers(0, 1 << 63, size=n, dtype=np.uint64) % np.uint64(P)).astype(np.uint64)
        out = np.zeros(4, dtype=np.uint64)
        L.dpo_hash_bases(v.ctypes.data_as(C.c_void_p), C.c_uint64(n), out.ctypes.data_as(C.c_void_p))
        assert out.tobytes() == blake3.blake3(v.astype("<u8").tobytes()).digest()          # hash_bases: LE canonical u64 bytes
    a = rng.integers(0, 1 << 63, size=4, dtype=np.uint64); b = rng.integers(0, 1 << 63, size=4, dtype=np.uint64)
    out = np.zeros(4, dtype=np.uint64)
    L.dpo_hash_two_digests(a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    assert out.tobytes() == blake3.blake3(a.tobytes() + b.tobytes()).digest()             # hash_two_digests: left || right


def test_merkle_root_of_a_small_tree_by_hand(blake_checker):
    """MerkleTree::from_leaves (mpcs/src/util/merkle_tree.rs:36-60,261-330) under BlakeHasher, recomputed with the Python package.
    A trivial commitment (num_vars <= 7) is the tree over the raw evaluations (basefold.rs:304-330)."""
    nv = 5
    ev = O.splitmix_f(77, 1 << nv)
    root, _, _ = O.pcs_commit(ev, False, 8)
    level = [blake3.blake3(ev[2 * i: 2 * i + 2].astype("<u8").tobytes()).digest() for i in range(len(ev) // 2)]
    while len(level) > 1:
        level = [blake3.blake3(level[2 * i] + level[2 * i + 1]).digest() for i in range(len(level) // 2)]
    assert root.tobytes() == level[0]


def test_proofs_verify_under_blake_and_differ_from_poseidon(blake_checker):
    nv = 10
    ev = O.splitmix_f(5, 1 << nv); pt = O.splitmix_e(6, nv)
    flat = O.pcs_open(ev, False, nv, pt)
    root = O.pcs_commit(ev, False, nv, want_codeword=False)[0]
    assert O.pcs_verify(flat, root, nv, True, nv, pt, O.evaluate(ev, False, pt)) is None
    bad = flat.copy(); bad[len(bad) // 2] ^= np.uint64(1)
    assert O.pcs_verify(bad, root, nv, True, nv, pt, O.evaluate(ev, False, pt)) is not None
    assert O.zkml_prove_verify(2, 32, 1, 2) is None
    O.set_hash_mode(0)
    assert not np.array_equal(O.pcs_commit(ev, False, nv, want_codeword=False)[0], root)
    assert O.pcs_verify(flat, root, nv, True, nv, pt, O.evaluate(ev, False, pt)) is not None      # a blake proof is rejected by the Poseidon verifier
