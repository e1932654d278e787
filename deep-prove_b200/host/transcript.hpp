// Host Fiat-Shamir: Poseidon2 width-8 permutation, duplex sponge, BasicTranscript.
// north_star keeps the transcript on the host; this is the host-language side of the boundary (the
// reference's `transcript` and `poseidon` crates), written in C++ because no Rust toolchain exists here.
// Reference: transcript/src/{lib.rs:22-93,basic.rs}, poseidon/src/challenger.rs:14-44,
// ff_ext/src/lib.rs:177-235.  Constants: include/dp_poseidon2_constants.h (provenance there).
#pragma once
#include "field.hpp"
#include "../../include/dp_poseidon2_constants.h"
#include "../../include/dp_blake3.h"
#include <cstring>
#include <stdexcept>

namespace dp {

class Poseidon2 {
  public:
    // The sponge sits on the critical path between device rounds (~3400 permutations per Dense-4M proof), so the permutation
    // is written like the device one (csrc/poseidon2.cuh): state words stay "weak" (any u64, not reduced below p), products
    // are reduced 128 -> 64 bits without canonicalising, the linear layers accumulate in 128 bits and fold once per output,
    // the internal layer's s[i] * diag[i] + sum is ONE reduction.  Exact modular arithmetic throughout; canonical in, canonical out.
    static void permute(u64 s[8]) {
        linear_ext(s);
        for (int r = 0; r < 4; r++) { for (int i = 0; i < 8; i++) s[i] = pow7(wadd(s[i], DP_P2_EXT_RC[0][r][i])); linear_ext(s); }
        for (int r = 0; r < 22; r++) {
            s[0] = pow7(wadd(s[0], DP_P2_INT_RC[r]));
            u128 tot = 0;
            for (int i = 0; i < 8; i++) tot += s[i];                                        // < 2^67
            for (int i = 0; i < 8; i++) s[i] = wred((u128)s[i] * DP_P2_DIAG[i] + tot);      // < 2^128 - 2^96 + 2^67: no overflow
        }
        for (int r = 0; r < 4; r++) { for (int i = 0; i < 8; i++) s[i] = pow7(wadd(s[i], DP_P2_EXT_RC[1][r][i])); linear_ext(s); }
        for (int i = 0; i < 8; i++) s[i] = canon(s[i]);
    }
    // the straightforward canonical formulation (kept as the cross-check of the fast path, tests/test_hash_transcript.py)
    static void permute_canonical(u64 s[8]) {
        linear_ext_c(s);
        for (int r = 0; r < 4; r++) { for (int i = 0; i < 8; i++) s[i] = pow7_c(fadd(s[i], DP_P2_EXT_RC[0][r][i])); linear_ext_c(s); }
        for (int r = 0; r < 22; r++) {
            s[0] = pow7_c(fadd(s[0], DP_P2_INT_RC[r]));
            u64 tot = 0;
            for (int i = 0; i < 8; i++) tot = fadd(tot, s[i]);
            for (int i = 0; i < 8; i++) s[i] = fadd(fmul(s[i], DP_P2_DIAG[i]), tot);
        }
        for (int r = 0; r < 4; r++) { for (int i = 0; i < 8; i++) s[i] = pow7_c(fadd(s[i], DP_P2_EXT_RC[1][r][i])); linear_ext_c(s); }
    }
  private:
    // hi * 2^64 + lo -> some representative in [0, 2^64): 2^64 = 2^32 - 1, 2^96 = -1 (mod p); branch-free
    static u64 wred(u128 x) {
        u64 lo = (u64)x, hi = (u64)(x >> 64), hh = hi >> 32, hl = hi & EPS;
        u64 t0 = lo - hh; t0 -= ((u64)0 - (u64)(lo < hh)) & EPS;
        u64 t1 = (hl << 32) - hl;
        u64 r = t0 + t1; r += ((u64)0 - (u64)(r < t1)) & EPS;
        return r;
    }
    static u64 wmul(u64 a, u64 b) { return wred((u128)a * b); }
    static u64 wadd(u64 a, u64 c) { u64 r = a + c; r += ((u64)0 - (u64)(r < a)) & EPS; return r; }   // a weak, c < p: at most one wrap, then + EPS cannot wrap again
    static u64 pow7(u64 x) { u64 a = wmul(x, x), b = wmul(a, a); return wmul(wmul(a, x), b); }
    // circ(2,3,1,1) on each half, then add the column sums (p3 MDSMat4 + mds_light_permutation): out[i] = 2 n[i] + n[i ^ 4], n < 7 * 2^64
    static void linear_ext(u64 *s) {
        u128 n[8];
        for (int h = 0; h < 8; h += 4) {
            const u64 *x = s + h;
            u128 a = (u128)x[0] + x[1], b = (u128)x[2] + x[3], all = a + b;
            n[h + 0] = all + x[1] + a;                 // 2 x0 + 3 x1 + x2 + x3
            n[h + 1] = all + x[1] + x[2] + x[2];       // x0 + 2 x1 + 3 x2 + x3
            n[h + 2] = all + x[3] + b;                 // x0 + x1 + 2 x2 + 3 x3
            n[h + 3] = all + x[3] + x[0] + x[0];       // 3 x0 + x1 + x2 + 2 x3
        }
        for (int i = 0; i < 8; i++) s[i] = wred(n[i] + n[i] + n[i ^ 4]);
    }
    static u64 pow7_c(u64 x) { u64 a = fmul(x, x), b = fmul(a, a); return fmul(fmul(a, x), b); }
    static void linear_ext_c(u64 *s) {
        for (int h = 0; h < 8; h += 4) {
            u64 *x = s + h;
            u64 a = fadd(x[0], x[1]), b = fadd(x[2], x[3]), all = fadd(a, b);
            u64 y0 = fadd(fadd(all, x[1]), a), y2 = fadd(fadd(all, x[3]), b);  // rows (2,3,1,1) and (1,1,2,3)
            u64 y1 = fadd(fadd(all, x[1]), fadd(x[2], x[2]));
            u64 y3 = fadd(fadd(all, x[3]), fadd(x[0], x[0]));
            x[0] = y0; x[1] = y1; x[2] = y2; x[3] = y3;
        }
        for (int k = 0; k < 4; k++) { u64 c = fadd(s[k], s[k + 4]); s[k] = fadd(s[k], c); s[k + 4] = fadd(s[k + 4], c); }
    }
};

// DuplexChallenger<F, Poseidon2, WIDTH = 8, RATE = 4>
class Sponge {
  public:
    Sponge() { memset(st_, 0, sizeof st_); memset(in_, 0, sizeof in_); memset(out_, 0, sizeof out_); }
    void observe(u64 v) {
        nout_ = 0;
        in_[nin_++] = v;
        if (nin_ == 4) duplex();
    }
    u64 sample() {
        if (nin_ || !nout_) duplex();
        return out_[--nout_];
    }
    // the whole state as 14 words [st[0..7], in[0..3], nin, nout] (dp_sc_run_tail_fs continues it on the device).  out is not
    // part of it: a duplex copies st[0..3] into it and nothing else changes st before the next duplex.
    static constexpr int WORDS = 14;
    void save(u64 w[WORDS]) const { memcpy(w, st_, 64); memcpy(w + 8, in_, 32); w[12] = (u64)nin_; w[13] = (u64)nout_; }
    void load(const u64 w[WORDS]) { memcpy(st_, w, 64); memcpy(in_, w + 8, 32); nin_ = (int)w[12]; nout_ = (int)w[13]; memcpy(out_, st_, 32); }
  private:
    void duplex() {
        for (int i = 0; i < nin_; i++) st_[i] = in_[i];
        nin_ = 0;
        Poseidon2::permute(st_);
        memcpy(out_, st_, 32); nout_ = 4;
    }
    u64 st_[8], in_[4], out_[4];
    int nin_ = 0, nout_ = 0;
};

// Which state a transcript hands to the device transcript of the resident kernels (save_sponge's result): none (the host runs every
// round), BasicTranscript's duplex sponge (Sponge::WORDS words, dp_sc_run_tail_fs / dp_logup_run_layers_fs) or BlakeTranscript's
// hasher image (dpb3::IMAGE_WORDS words, the _blake entry points).  A buffer of DEVICE_STATE_WORDS holds either.
enum DeviceState : int { DS_NONE = 0, DS_POSEIDON2 = 1, DS_BLAKE3 = 2 };
static constexpr size_t DEVICE_STATE_WORDS = dpb3::IMAGE_WORDS;
static_assert(DEVICE_STATE_WORDS >= (size_t)Sponge::WORDS, "the state buffer holds the Poseidon2 sponge too");

// trait Transcript<E> as implemented by BasicTranscript<E>
class BasicTranscript {
  public:
    explicit BasicTranscript(const std::string &label) { append_message(label); }
    void append_field_element(u64 f) { sp_.observe(canon(f)); }
    void append_field_elements(const std::vector<u64> &f) { for (u64 x : f) append_field_element(x); }
    void append_message(const uint8_t *m, size_t n) {
        for (size_t i = 0; i < n; i += 8) { u64 v = 0; memcpy(&v, m + i, n - i < 8 ? n - i : 8); sp_.observe(v); }
    }
    void append_message(const std::string &s) { append_message((const uint8_t *)s.data(), s.size()); }
    void append_usize(u64 v) { sp_.observe(v); }  // usize::to_le_bytes() -> one field element
    void append_field_element_ext(const Ext &e) { sp_.observe(e.c0); sp_.observe(e.c1); }
    void append_field_element_exts(const ExtVec &v) { for (auto &e : v) append_field_element_ext(e); }
    Ext read_challenge() { u64 a = sp_.sample(); u64 b = sp_.sample(); return Ext(a, b); }
    Ext get_and_append_challenge(const std::string &label) { append_message(label); return read_challenge(); }
    // the sponge state for dp_sc_run_tail_fs: this transcript can always continue on the device
    int save_sponge(u64 w[Sponge::WORDS]) const { sp_.save(w); return DS_POSEIDON2; }
    void load_sponge(const u64 w[Sponge::WORDS]) { sp_.load(w); }
  private:
    Sponge sp_;
};

// BlakeTranscript (transcript/src/blake.rs), the transcript of the reference's `blake` feature (zkml/src/bin/bench.rs:29-44): one running
// BLAKE3 hasher.  Through trait Transcript<E> (transcript/src/lib.rs:22-93) a base element is absorbed as update("field_element") +
// update(BigUint::to_bytes_le of the canonical value: no trailing zero bytes, [0] for zero); an extension element as
// update("field_element_ext") + update(bytes(c0) || bytes(c1)); a message goes through the trait default (8-byte chunks -> field
// elements -> one append each); a challenge is update("challenge") + 16 bytes of finalize_xof read as two little-endian u64, retried
// until both are canonical (ff_ext/src/lib.rs:29-41,246-254).  BLAKE3 itself: include/dp_blake3.h (pinned against the Python package).
class BlakeTranscript {
  public:
    explicit BlakeTranscript(const std::string &label) { h_.update(label.data(), label.size()); }   // BlakeTranscript::new: raw label bytes
    void append_field_element(u64 f) { uint8_t b[8]; size_t n = le(canon(f), b); h_.update("field_element", 13); h_.update(b, n); }
    void append_field_elements(const std::vector<u64> &f) { for (u64 x : f) append_field_element(x); }
    void append_message(const uint8_t *m, size_t n) { for (size_t i = 0; i < n; i += 8) { u64 v = 0; memcpy(&v, m + i, n - i < 8 ? n - i : 8); append_field_element(v); } }
    void append_message(const std::string &s) { append_message((const uint8_t *)s.data(), s.size()); }
    void append_usize(u64 v) { append_field_element(v); }
    void append_field_element_ext(const Ext &e) { uint8_t b[16]; size_t n0 = le(canon(e.c0), b), n1 = le(canon(e.c1), b + n0); h_.update("field_element_ext", 17); h_.update(b, n0 + n1); }
    void append_field_element_exts(const ExtVec &v) { for (auto &e : v) append_field_element_ext(e); }
    Ext read_challenge() {
        for (;;) {
            h_.update("challenge", 9);
            uint8_t o[16]; h_.finalize(o, 16);
            u64 a, b; memcpy(&a, o, 8); memcpy(&b, o + 8, 8);
            if (a < P && b < P) return Ext(a, b);
        }
    }
    Ext get_and_append_challenge(const std::string &label) { append_message(label); return read_challenge(); }
    // the hasher image for the _blake device entry points; none (the host keeps every round) past 2^16 absorbed chunks
    int save_sponge(u64 w[dpb3::IMAGE_WORDS]) const { return h_.save(w) ? DS_BLAKE3 : DS_NONE; }
    void load_sponge(const u64 w[dpb3::IMAGE_WORDS]) {
        if (!dpb3::image_ok(w)) throw std::invalid_argument("BlakeTranscript::load_sponge: not a BLAKE3 hasher state");
        h_.load(w);
    }
  private:
    static size_t le(u64 c, uint8_t b[8]) { size_t n = 0; for (int k = 0; k < 8; k++) { b[k] = (uint8_t)(c >> (8 * k)); if (b[k]) n = k + 1; } return n ? n : 1; }
    dpb3::Hasher h_;
};

// The transcript the C entry points of the host library build: BasicTranscript, or BlakeTranscript after dph_set_hasher(1)
inline int &hasher_mode() { static int m = 0; return m; }
class DynTranscript {
  public:
    explicit DynTranscript(const std::string &label) : blake_(hasher_mode() == 1), b_(blake_ ? std::string() : label), k_(blake_ ? label : std::string()) {}
    void append_field_element(u64 f) { blake_ ? k_.append_field_element(f) : b_.append_field_element(f); }
    void append_field_elements(const std::vector<u64> &f) { for (u64 x : f) append_field_element(x); }
    void append_message(const uint8_t *m, size_t n) { blake_ ? k_.append_message(m, n) : b_.append_message(m, n); }
    void append_message(const std::string &s) { append_message((const uint8_t *)s.data(), s.size()); }
    void append_usize(u64 v) { blake_ ? k_.append_usize(v) : b_.append_usize(v); }
    void append_field_element_ext(const Ext &e) { blake_ ? k_.append_field_element_ext(e) : b_.append_field_element_ext(e); }
    void append_field_element_exts(const ExtVec &v) { for (auto &e : v) append_field_element_ext(e); }
    Ext read_challenge() { return blake_ ? k_.read_challenge() : b_.read_challenge(); }
    Ext get_and_append_challenge(const std::string &label) { append_message(label); return read_challenge(); }
    // w: DEVICE_STATE_WORDS; returns which state it holds (DeviceState)
    int save_sponge(u64 *w) const { return blake_ ? k_.save_sponge(w) : b_.save_sponge(w); }
    int state_kind() const { return blake_ ? DS_BLAKE3 : DS_POSEIDON2; }          // what load_sponge takes
    void load_sponge(const u64 *w) { blake_ ? k_.load_sponge(w) : b_.load_sponge(w); }
  private:
    bool blake_; BasicTranscript b_; BlakeTranscript k_;
};

}  // namespace dp
