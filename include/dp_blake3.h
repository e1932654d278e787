/* BLAKE3 (unkeyed hash mode) -- a small portable implementation of the published algorithm (the BLAKE3 paper, section 2;
 * same structure as the official reference_impl): incremental update, non-destructive finalize, extendable output.
 * Used by the `blake` variant of the path (mpcs/src/util/hash.rs:79-95 BlakeHasher, transcript/src/blake.rs BlakeTranscript),
 * which -- unlike the Poseidon2 variant -- is fully determined by the reference's own sources plus this standard primitive,
 * so it can be PINNED: tests/test_blake.py checks this file against the Python `blake3` package on many lengths, offsets and
 * output sizes.  Header-only, host code (the device has its own compression and incremental hasher in csrc/blake3.cuh; Hasher::save /
 * load exchange the state with it). */
#ifndef DP_BLAKE3_H
#define DP_BLAKE3_H
#include <stdint.h>
#include <string.h>
#include <stddef.h>

namespace dpb3 {

static const uint32_t IV[8] = {0x6A09E667, 0xBB67AE85, 0x3C6EF372, 0xA54FF53A, 0x510E527F, 0x9B05688C, 0x1F83D9AB, 0x5BE0CD19};
static const uint8_t MSG_PERM[16] = {2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8};
enum : uint32_t { CHUNK_START = 1, CHUNK_END = 2, PARENT = 4, ROOT = 8 };
static const size_t BLOCK_LEN = 64, CHUNK_LEN = 1024;

static inline uint32_t rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }
static inline void g(uint32_t *s, int a, int b, int c, int d, uint32_t mx, uint32_t my) {
    s[a] = s[a] + s[b] + mx; s[d] = rotr(s[d] ^ s[a], 16);
    s[c] = s[c] + s[d];      s[b] = rotr(s[b] ^ s[c], 12);
    s[a] = s[a] + s[b] + my; s[d] = rotr(s[d] ^ s[a], 8);
    s[c] = s[c] + s[d];      s[b] = rotr(s[b] ^ s[c], 7);
}
/* the compression function: 16 output words (the first 8 are the chaining value) */
static inline void compress(const uint32_t cv[8], const uint32_t block[16], uint64_t counter, uint32_t block_len, uint32_t flags, uint32_t out[16]) {
    uint32_t s[16] = {cv[0], cv[1], cv[2], cv[3], cv[4], cv[5], cv[6], cv[7], IV[0], IV[1], IV[2], IV[3], (uint32_t)counter, (uint32_t)(counter >> 32), block_len, flags};
    uint32_t m[16]; memcpy(m, block, 64);
    for (int r = 0; r < 7; r++) {
        g(s, 0, 4, 8, 12, m[0], m[1]);  g(s, 1, 5, 9, 13, m[2], m[3]);  g(s, 2, 6, 10, 14, m[4], m[5]);   g(s, 3, 7, 11, 15, m[6], m[7]);
        g(s, 0, 5, 10, 15, m[8], m[9]); g(s, 1, 6, 11, 12, m[10], m[11]); g(s, 2, 7, 8, 13, m[12], m[13]); g(s, 3, 4, 9, 14, m[14], m[15]);
        if (r < 6) { uint32_t t[16]; for (int i = 0; i < 16; i++) t[i] = m[MSG_PERM[i]]; memcpy(m, t, 64); }
    }
    for (int i = 0; i < 8; i++) { out[i] = s[i] ^ s[i + 8]; out[i + 8] = s[i + 8] ^ cv[i]; }
}
static inline void words_from_le(const uint8_t *b, size_t n, uint32_t w[16]) {   /* n <= 64 bytes, zero-padded */
    uint8_t tmp[64]; memset(tmp, 0, 64); memcpy(tmp, b, n);
    for (int i = 0; i < 16; i++) w[i] = (uint32_t)tmp[4 * i] | ((uint32_t)tmp[4 * i + 1] << 8) | ((uint32_t)tmp[4 * i + 2] << 16) | ((uint32_t)tmp[4 * i + 3] << 24);
}

/* what is needed to produce output: either a chunk's last block or a parent node */
struct Output {
    uint32_t cv[8], block[16]; uint64_t counter; uint32_t block_len, flags;
    void chaining_value(uint32_t out[8]) const { uint32_t o[16]; compress(cv, block, counter, block_len, flags, o); memcpy(out, o, 32); }
    void root_bytes(uint8_t *out, size_t n) const {       /* extendable output: block t of the stream = compress(..., counter = t, ROOT) */
        uint64_t t = 0; size_t off = 0;
        while (off < n) {
            uint32_t o[16]; compress(cv, block, t, block_len, flags | ROOT, o);
            for (int i = 0; i < 16 && off < n; i++) for (int k = 0; k < 4 && off < n; k++) out[off++] = (uint8_t)(o[i] >> (8 * k));
            t++;
        }
    }
};
struct ChunkState {
    uint32_t cv[8]; uint64_t chunk_counter; uint8_t block[64]; uint8_t block_len, blocks_compressed; uint32_t flags;
    void init(const uint32_t key[8], uint64_t counter, uint32_t fl) { memcpy(cv, key, 32); chunk_counter = counter; memset(block, 0, 64); block_len = 0; blocks_compressed = 0; flags = fl; }
    size_t len() const { return BLOCK_LEN * blocks_compressed + block_len; }
    uint32_t start_flag() const { return blocks_compressed == 0 ? CHUNK_START : 0; }
    void update(const uint8_t *in, size_t n) {
        while (n > 0) {
            if (block_len == BLOCK_LEN) {   /* the buffered block is not the last one of the chunk: compress it */
                uint32_t w[16], o[16]; words_from_le(block, 64, w);
                compress(cv, w, chunk_counter, (uint32_t)BLOCK_LEN, flags | start_flag(), o); memcpy(cv, o, 32);
                blocks_compressed++; memset(block, 0, 64); block_len = 0;
            }
            size_t take = BLOCK_LEN - block_len; if (take > n) take = n;
            memcpy(block + block_len, in, take); block_len += (uint8_t)take; in += take; n -= take;
        }
    }
    Output output() const { Output o; memcpy(o.cv, cv, 32); words_from_le(block, block_len, o.block); o.counter = chunk_counter; o.block_len = block_len; o.flags = flags | start_flag() | CHUNK_END; return o; }
};
static inline Output parent_output(const uint32_t l[8], const uint32_t r[8], const uint32_t key[8], uint32_t flags) {
    Output o; memcpy(o.cv, key, 32); memcpy(o.block, l, 32); memcpy(o.block + 8, r, 32); o.counter = 0; o.block_len = (uint32_t)BLOCK_LEN; o.flags = PARENT | flags; return o;
}

/* The hasher's state as IMAGE_WORDS u64 words -- the image a BlakeTranscript hands to the device (include/deepprove_b200.h,
 * DP_B3T_WORDS): [0..3] chunk chaining value (8 x u32, little-endian pairs), [4] chunk_counter, [5..12] the 64-byte block buffer,
 * [13] block_len, [14] blocks_compressed, [15] stack_len, [16 + 4i .. 19 + 4i] stack entry i.  Unkeyed hashing only (key = IV,
 * no mode flags).  image_ok: the image is one a Hasher can be in. */
static const size_t IMAGE_STACK = 16, IMAGE_WORDS = 16 + 4 * IMAGE_STACK;
static inline bool image_ok(const uint64_t *w) {
    if (w[13] > BLOCK_LEN || w[14] > 15 || (w[14] > 0 && w[13] == 0) || w[15] > IMAGE_STACK || w[15] != (uint64_t)__builtin_popcountll(w[4])) return false;
    for (size_t i = (size_t)w[13]; i < BLOCK_LEN; i++) if ((uint8_t)(w[5 + i / 8] >> (8 * (i % 8))) != 0) return false;
    return true;
}

class Hasher {
  public:
    Hasher() { memcpy(key_, IV, 32); chunk_.init(key_, 0, 0); stack_len_ = 0; }
    /* false (nothing written) when the stack is deeper than IMAGE_STACK: more than 2^16 chunks absorbed */
    bool save(uint64_t *w) const {
        if (stack_len_ > IMAGE_STACK) return false;
        memset(w, 0, 8 * IMAGE_WORDS);
        put8(w, chunk_.cv); w[4] = chunk_.chunk_counter;
        for (int i = 0; i < 64; i++) w[5 + i / 8] |= (uint64_t)chunk_.block[i] << (8 * (i % 8));
        w[13] = chunk_.block_len; w[14] = chunk_.blocks_compressed; w[15] = stack_len_;
        for (size_t i = 0; i < stack_len_; i++) put8(w + 16 + 4 * i, stack_[i]);
        return true;
    }
    /* an image that passes image_ok */
    void load(const uint64_t *w) {
        memcpy(key_, IV, 32); chunk_.init(key_, w[4], 0);
        get8(w, chunk_.cv);
        for (int i = 0; i < 64; i++) chunk_.block[i] = (uint8_t)(w[5 + i / 8] >> (8 * (i % 8)));
        chunk_.block_len = (uint8_t)w[13]; chunk_.blocks_compressed = (uint8_t)w[14]; stack_len_ = (size_t)w[15];
        for (size_t i = 0; i < stack_len_; i++) get8(w + 16 + 4 * i, stack_[i]);
    }
    void update(const void *data, size_t n) {
        const uint8_t *in = (const uint8_t *)data;
        while (n > 0) {
            if (chunk_.len() == CHUNK_LEN) {   /* chunk complete and more input follows: push its chaining value, merging completed subtrees */
                uint32_t cv[8]; chunk_.output().chaining_value(cv);
                uint64_t total = chunk_.chunk_counter + 1;
                add_chunk_cv(cv, total);
                chunk_.init(key_, total, 0);
            }
            size_t want = CHUNK_LEN - chunk_.len(); if (want > n) want = n;
            chunk_.update(in, want); in += want; n -= want;
        }
    }
    /* non-destructive: the hasher can keep absorbing afterwards (blake3::Hasher::finalize / finalize_xof) */
    void finalize(uint8_t *out, size_t n) const {
        Output o = chunk_.output();
        for (int i = (int)stack_len_ - 1; i >= 0; i--) { uint32_t cv[8]; o.chaining_value(cv); o = parent_output(stack_[i], cv, key_, 0); }
        o.root_bytes(out, n);
    }
  private:
    static void put8(uint64_t *w, const uint32_t v[8]) { for (int k = 0; k < 4; k++) w[k] = (uint64_t)v[2 * k] | ((uint64_t)v[2 * k + 1] << 32); }
    static void get8(const uint64_t *w, uint32_t v[8]) { for (int k = 0; k < 4; k++) { v[2 * k] = (uint32_t)w[k]; v[2 * k + 1] = (uint32_t)(w[k] >> 32); } }
    void add_chunk_cv(uint32_t cv[8], uint64_t total_chunks) {
        while ((total_chunks & 1) == 0) {   /* one merge per trailing zero bit of the chunk count */
            uint32_t p[8]; parent_output(stack_[stack_len_ - 1], cv, key_, 0).chaining_value(p); memcpy(cv, p, 32); stack_len_--; total_chunks >>= 1;
        }
        memcpy(stack_[stack_len_++], cv, 32);
    }
    uint32_t key_[8]; ChunkState chunk_; uint32_t stack_[54][8]; size_t stack_len_;
};
static inline void hash(const void *data, size_t n, uint8_t out[32]) { Hasher h; h.update(data, n); h.finalize(out, 32); }

}  // namespace dpb3
#endif
