#!/usr/bin/env python3
"""Regenerates tests/golden/blake_retry.json: a BlakeTranscript state from which the first challenge of a sumcheck draws a limb >= p,
so read_challenge has to retry (tests/test_gpu_blake_device_transcript.py::test_retry_path).

A challenge's 16 output bytes hold a non-canonical limb with probability about 2^-31, so such a state has to be searched for.  The
transcript is BlakeTranscript::new(label) with a label of 1024 + 16 bytes whose first chunk ends in a 16-hex-digit nonce.  The
sumcheck (the MLEs and product below, nv = 4, max_degree = 2) starts right after it; its round-0 message depends on no challenge, so
the bytes of round 0 -- the message, the label "Internal round", "challenge" -- are fixed.  For each nonce the search needs two
BLAKE3 compressions: the last block of chunk 0, and the ROOT parent node over the two chunks (the second chunk's chaining value does
not depend on the nonce).  It runs a small C++ program over include/dp_blake3.h on every core: about 2^31 nonces on average, four
minutes on an 8-core host.  The result is checked with the Python `blake3` package before it is written.  Run from the repository root:
    python tests/golden/make_blake_retry.py
"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_py as O  # noqa: E402
import blake3  # noqa: E402

P = O.P
NV, MAX_DEG = 4, 2
MLES = [(5, True), (6, False)]                  # (splitmix seed, extension field) of 2^NV entries each
PRODUCT = ((3, 4), [0, 1])                      # coefficient, MLE indices
HEAD = bytes((ord("a") + i % 26) for i in range(1008))   # chunk 0 before the nonce
TAIL = b"handed over here"                      # 16 bytes of chunk 1 before the sumcheck


def mles():
    return [(O.splitmix_e(s, 1 << NV) if ext else O.splitmix_f(s, 1 << NV), ext) for s, ext in MLES]


def fe(v):
    v %= P
    return v.to_bytes(8, "little").rstrip(b"\0") or b"\0"


def round0_bytes():
    """what BlakeTranscript absorbs in round 0 up to the first finalize"""
    msgs, _ = O.sumcheck_rounds_fixed(mles(), [PRODUCT], NV, [[0, 0]] * NV)
    out = b"".join(b"field_element_ext" + fe(int(c0)) + fe(int(c1)) for c0, c1 in msgs[0])
    for w in (b"Internal", b" round"):
        out += b"field_element" + fe(int.from_bytes(w, "little"))
    return out + b"challenge"


SEARCH = r"""
#include "dp_blake3.h"
#include <atomic>
#include <cstdio>
#include <string>
#include <thread>
#include <vector>
using namespace dpb3;
static const uint64_t P = 0xFFFFFFFF00000001ULL;
int main(int argc, char **argv) {
    std::string head, tail;   // hex on the command line
    auto unhex = [](const char *h) { std::string s; for (size_t i = 0; h[i] && h[i + 1]; i += 2) s.push_back((char)std::stoi(std::string(h + i, 2), nullptr, 16)); return s; };
    head = unhex(argv[1]); tail = unhex(argv[2]);
    uint32_t cv15[8]; memcpy(cv15, IV, 32);
    for (int b = 0; b < 15; b++) { uint32_t w[16], o[16]; words_from_le((const uint8_t *)head.data() + 64 * b, 64, w); compress(cv15, w, 0, 64, b == 0 ? CHUNK_START : 0, o); memcpy(cv15, o, 32); }
    ChunkState c1; c1.init(IV, 1, 0); c1.update((const uint8_t *)tail.data(), tail.size());
    uint32_t cv1[8]; c1.output().chaining_value(cv1);
    std::atomic<bool> found(false); std::atomic<uint64_t> result(0);
    const unsigned T = std::thread::hardware_concurrency();
    std::vector<std::thread> th;
    for (unsigned t = 0; t < T; t++) th.emplace_back([&, t] {
        uint8_t last[64]; memcpy(last, head.data() + 960, 48);
        for (uint64_t n = t; !found.load(std::memory_order_relaxed); n += T) {
            for (int k = 0; k < 16; k++) last[48 + k] = "0123456789abcdef"[(n >> (60 - 4 * k)) & 15];
            uint32_t w[16], o[16], cv0[8]; words_from_le(last, 64, w);
            compress(cv15, w, 0, 64, CHUNK_END, o); memcpy(cv0, o, 32);
            memcpy(w, cv0, 32); memcpy(w + 8, cv1, 32);
            compress(IV, w, 0, 64, PARENT | ROOT, o);
            const uint64_t a = (uint64_t)o[0] | ((uint64_t)o[1] << 32), b = (uint64_t)o[2] | ((uint64_t)o[3] << 32);
            if (a >= P || b >= P) { if (!found.exchange(true)) result = n; }
        }
    });
    for (auto &x : th) x.join();
    printf("%016llx\n", (unsigned long long)result.load());
    return 0;
}
"""


def main():
    r0 = round0_bytes()
    assert len(TAIL) + len(r0) <= 1024, "round 0 stays in chunk 1"
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "search.cpp"), os.path.join(d, "search")
        open(src, "w").write(SEARCH)
        subprocess.check_call(["g++", "-O3", "-march=native", "-std=c++17", "-pthread", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        nonce = subprocess.check_output([exe, HEAD.hex(), (TAIL + r0).hex()]).decode().strip()
    label = HEAD + nonce.encode() + TAIL
    o = blake3.blake3(label + r0).digest(length=16)
    a, b = int.from_bytes(o[:8], "little"), int.from_bytes(o[8:], "little")
    assert a >= P or b >= P, "the search result does not retry"
    out = {"label": label.decode(), "nv": NV, "max_deg": MAX_DEG, "mles": MLES, "product": [list(PRODUCT[0]), PRODUCT[1]],
           "first_attempt": [a, b]}
    with open(os.path.join(HERE, "blake_retry.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("nonce", nonce, "first attempt", hex(a), hex(b))


if __name__ == "__main__":
    main()
