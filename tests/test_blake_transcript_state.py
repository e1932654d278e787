"""The state image of a BlakeTranscript (include/dp_blake3.h Hasher::save / load, host/transcript.hpp BlakeTranscript::save_sponge):
the DP_B3T_WORDS words a prover hands to the device transcript (dp_sc_run_tail_fs_blake, dp_logup_run_layers_fs_blake).  A
transcript saved after any prefix and loaded into a fresh one continues exactly as the Python `blake3` package does, the image
follows blake3::Hasher's lazy rules, a transcript of more than 2^16 chunks has no image, and load refuses images no hasher can be in."""
import numpy as np
import pytest

blake3 = pytest.importorskip("blake3")
import test_blake as TB  # noqa: E402

P = TB.P
WORDS = 80
# prefixes: stack lengths 0 to 6, a pending full block (64), a full chunk not yet pushed (1024, 2048), a fresh block (65, 1025)
PREFIXES = [0, 1, 63, 64, 65, 1023, 1024, 1025, 2047, 2048, 3072] + [4096 * k for k in (1, 2, 3, 4, 5, 31)]


def _label(n):
    return ((np.arange(n, dtype=np.uint64) * 7) % 255 + 1).astype(np.uint8).tobytes()    # no zero byte: it travels as a C string


@pytest.fixture()
def host():
    import dpb200 as dp
    dp.set_hasher(1)
    yield dp
    dp.set_hasher(0)


def _expected_image_fields(n):
    """chunk_counter, block_len, blocks_compressed, stack_len of blake3::Hasher after n bytes (lazy: nothing is compressed until
    more input follows)"""
    pushed = (n - 1) // 1024 if n else 0
    in_chunk = n - 1024 * pushed
    nb = (in_chunk - 1) // 64 if in_chunk else 0
    return pushed, in_chunk - 64 * nb, nb, bin(pushed).count("1")


@pytest.mark.parametrize("n", PREFIXES)
def test_saved_state_continues_like_the_package(host, n):
    label = _label(n)
    t = host.Transcript(label)
    try:
        kind, w = t.save_state()
    finally:
        t.free()
    assert kind == 2
    ctr, blen, nblk, slen = _expected_image_fields(n)
    assert [int(w[4]), int(w[13]), int(w[14]), int(w[15])] == [ctr, blen, nblk, slen]
    block = w[5:13].tobytes()
    assert block[:blen] == label[n - blen:n] and block[blen:] == b"\0" * (64 - blen)
    assert not w[16 + 4 * slen:].any()
    fresh = host.Transcript(b"something else")
    try:
        fresh.load_state(2, w)
        got = TB._script(lambda _: fresh, *TB.host_transcript_ops())
        kind2, w2 = fresh.save_state()
    finally:
        fresh.free()
    py = TB._script(lambda _: TB.PyBlakeTranscript(label), lambda t, f: [t.append_f(x) for x in f], lambda t, m: t.append_msg(m),
                    lambda t, e: [t.append_e(*x) for x in e], lambda t, lbl: t.challenge(lbl), lambda t: t.read_challenge())
    assert got == py
    assert kind2 == 2 and int(w2[4]) >= ctr


def test_sixteen_stack_entries_save_and_seventeen_refuse(host):
    """2^16 - 1 pushed chunks: 16 stack entries, the deepest image; 2^17 - 1: 17 entries, no image (the host keeps the transcript)"""
    n16 = (2 ** 16 - 1) * 1024 + 1
    label = _label(n16)
    t = host.Transcript(label)
    try:
        kind, w = t.save_state()
        assert kind == 2 and int(w[15]) == 16 and int(w[4]) == 2 ** 16 - 1
        fresh = host.Transcript(b"")
        try:
            fresh.load_state(2, w)
            got = TB._script(lambda _: fresh, *TB.host_transcript_ops())
        finally:
            fresh.free()
    finally:
        t.free()
    py = TB._script(lambda _: TB.PyBlakeTranscript(label), lambda t, f: [t.append_f(x) for x in f], lambda t, m: t.append_msg(m),
                    lambda t, e: [t.append_e(*x) for x in e], lambda t, lbl: t.challenge(lbl), lambda t: t.read_challenge())
    assert got == py
    t = host.Transcript(_label((2 ** 17 - 1) * 1024 + 1))
    try:
        kind, w = t.save_state()
    finally:
        t.free()
    assert kind == 0


def malformed_images():
    """(name, image) for every rule an image must satisfy, each broken once from a valid image after 2100 bytes"""
    ok = np.zeros(WORDS, dtype=np.uint64)
    ok[4] = 2; ok[13] = 52; ok[14] = 0; ok[15] = 1; ok[5] = 0x0101010101010101
    out = []
    w = ok.copy(); w[13] = 65; out.append(("block_len_above_64", w))
    w = ok.copy(); w[14] = 16; out.append(("blocks_compressed_above_15", w))
    w = ok.copy(); w[14] = 3; w[13] = 0; w[5] = 0; out.append(("compressed_blocks_with_an_empty_buffer", w))
    w = ok.copy(); w[12] = 1 << 56; out.append(("byte_past_block_len", w))
    w = ok.copy(); w[15] = 2; out.append(("stack_len_not_popcount", w))
    w = ok.copy(); w[4] = (1 << 17) - 1; w[15] = 17; out.append(("stack_deeper_than_16", w))
    return ok, out


def test_load_refuses_malformed_images(host):
    ok, bad = malformed_images()
    t = host.Transcript(b"x")
    try:
        t.load_state(2, ok)
        for name, w in bad:
            try:
                t.load_state(2, w)
            except host.DpError:
                continue
            pytest.fail("a malformed image was loaded: " + name)
        with pytest.raises(host.DpError):         # a Poseidon2 state into a BLAKE3 transcript
            t.load_state(1, ok)
    finally:
        t.free()
