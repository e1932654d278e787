// BLAKE3 compression on the device for the `blake` Merkle hasher (mpcs/src/util/hash.rs:79-95 BlakeHasher): every hash this path
// needs is a single chunk -- a leaf pair (16 or 32 bytes), two digests (64 bytes), or the values of all polynomials of a batch
// commitment at one index (<= 1024 bytes).  State in registers, message schedule resolved at compile time.  Below it, the
// incremental hasher and the framing of BlakeTranscript that the resident sumcheck kernels run (csrc/sumcheck.cu TrB3).
// The algorithm is the published BLAKE3 (host twin: include/dp_blake3.h, pinned against the Python `blake3` package).
#pragma once
#include "gl.cuh"

namespace b3 {
enum : u32 { CHUNK_START = 1, CHUNK_END = 2, PARENT = 4, ROOT = 8 };
__device__ __forceinline__ u32 rotr(u32 x, int n) { return __funnelshift_r(x, x, n); }
__device__ __forceinline__ void g(u32 &a, u32 &b, u32 &c, u32 &d, u32 mx, u32 my) {
    a = a + b + mx; d = rotr(d ^ a, 16); c = c + d; b = rotr(b ^ c, 12);
    a = a + b + my; d = rotr(d ^ a, 8);  c = c + d; b = rotr(b ^ c, 7);
}
// message word order of round r = the permutation (2 6 3 10 7 0 4 13 1 11 12 5 9 14 15 8) applied r times
__device__ __forceinline__ constexpr int sched(int r, int i) {
    constexpr int P[16] = {2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8};
    int k = i; for (int t = 0; t < r; t++) k = P[k]; return k;
}
template <int R> __device__ __forceinline__ void round_fn(u32 (&s)[16], const u32 (&m)[16]) {
    g(s[0], s[4], s[8], s[12], m[sched(R, 0)], m[sched(R, 1)]);   g(s[1], s[5], s[9], s[13], m[sched(R, 2)], m[sched(R, 3)]);
    g(s[2], s[6], s[10], s[14], m[sched(R, 4)], m[sched(R, 5)]);  g(s[3], s[7], s[11], s[15], m[sched(R, 6)], m[sched(R, 7)]);
    g(s[0], s[5], s[10], s[15], m[sched(R, 8)], m[sched(R, 9)]);  g(s[1], s[6], s[11], s[12], m[sched(R, 10)], m[sched(R, 11)]);
    g(s[2], s[7], s[8], s[13], m[sched(R, 12)], m[sched(R, 13)]); g(s[3], s[4], s[9], s[14], m[sched(R, 14)], m[sched(R, 15)]);
}
// chaining value of one block at chunk `counter` (also the first 32 bytes of a ROOT block's output at output counter 0)
__device__ __forceinline__ void compress_ctr(u32 (&cv)[8], const u32 (&m)[16], u64 counter, u32 block_len, u32 flags) {
    u32 s[16] = {cv[0], cv[1], cv[2], cv[3], cv[4], cv[5], cv[6], cv[7], 0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au,
                 (u32)counter, (u32)(counter >> 32), block_len, flags};
    round_fn<0>(s, m); round_fn<1>(s, m); round_fn<2>(s, m); round_fn<3>(s, m); round_fn<4>(s, m); round_fn<5>(s, m); round_fn<6>(s, m);
#pragma unroll
    for (int i = 0; i < 8; i++) cv[i] = s[i] ^ s[i + 8];
}
// counter 0: every Merkle hash here is a single chunk
__device__ __forceinline__ void compress(u32 (&cv)[8], const u32 (&m)[16], u32 block_len, u32 flags) { compress_ctr(cv, m, 0ULL, block_len, flags); }
__device__ __forceinline__ void iv(u32 (&cv)[8]) {
    cv[0] = 0x6A09E667u; cv[1] = 0xBB67AE85u; cv[2] = 0x3C6EF372u; cv[3] = 0xA54FF53Au; cv[4] = 0x510E527Fu; cv[5] = 0x9B05688Cu; cv[6] = 0x1F83D9ABu; cv[7] = 0x5BE0CD19u;
}
__device__ __forceinline__ void put(u32 (&m)[16], int k, u64 v) { m[2 * k] = (u32)v; m[2 * k + 1] = (u32)(v >> 32); }
__device__ __forceinline__ void digest_words(const u32 (&cv)[8], u64 out[4]) {
#pragma unroll
    for (int k = 0; k < 4; k++) out[k] = (u64)cv[2 * k] | ((u64)cv[2 * k + 1] << 32);
}
// BLAKE3 of nw u64 words (nw <= 8: one block), little-endian
__device__ __forceinline__ void hash_words(const u64 *w, int nw, u64 out[4]) {
    u32 m[16];
#pragma unroll
    for (int k = 0; k < 8; k++) put(m, k, k < nw ? w[k] : 0ULL);
    u32 cv[8]; iv(cv);
    compress(cv, m, 8u * nw, CHUNK_START | CHUNK_END | ROOT);
    digest_words(cv, out);
}
// BLAKE3 of n u64 words fetched through get(i), n <= 128 (one chunk of up to 16 blocks)
template <class F> __device__ __forceinline__ void hash_stream(F get, int n, u64 out[4]) {
    u32 cv[8]; iv(cv);
    const int nblocks = n == 0 ? 1 : (n + 7) / 8;
    for (int b = 0; b < nblocks; b++) {
        u32 m[16];
#pragma unroll
        for (int k = 0; k < 8; k++) put(m, k, 8 * b + k < n ? get(8 * b + k) : 0ULL);
        const int words = n - 8 * b < 8 ? n - 8 * b : 8;
        compress(cv, m, 8u * (u32)words, (b == 0 ? CHUNK_START : 0u) | (b == nblocks - 1 ? (CHUNK_END | ROOT) : 0u));
    }
    digest_words(cv, out);
}

// ---- incremental hasher over a state image (BlakeTranscript on the device) --------------------------------------------------------
// blake3::Hasher, unkeyed, on the DP_B3T_WORDS image of include/deepprove_b200.h (dpb3::Hasher::save / load): [0..3] chunk chaining
// value, [4] chunk_counter, [5..12] block buffer (zero past block_len), [13] block_len, [14] blocks_compressed, [15] stack_len,
// [16 + 4i ..] stack entry i.  One thread works on the image in place (shared memory in the resident kernels).  absorb follows the
// lazy rules of dpb3::Hasher::update exactly -- a full block is compressed, and a full chunk pushed and merged once per trailing zero
// bit of the new chunk count, only when more input arrives -- so after any byte stream the image equals the host's.
enum : int { T_CV = 0, T_CTR = 4, T_BLOCK = 5, T_BLEN = 13, T_NBLK = 14, T_SLEN = 15, T_STACK = 16, T_STACK_MAX = 16 };
static constexpr u64 T_OVERFLOW = 1ULL << 32;   // set in word T_SLEN when a push found the stack full (the image is then unusable)
__device__ __forceinline__ void t_get(const u64 *w, u32 (&v)[8]) {
#pragma unroll
    for (int k = 0; k < 4; k++) { v[2 * k] = (u32)w[k]; v[2 * k + 1] = (u32)(w[k] >> 32); }
}
__device__ __forceinline__ void t_put(u64 *w, const u32 (&v)[8]) {
#pragma unroll
    for (int k = 0; k < 4; k++) w[k] = (u64)v[2 * k] | ((u64)v[2 * k + 1] << 32);
}
// the n <= 8 low bytes of x, little-endian
static __device__ __noinline__ void t_absorb(u64 *w, u64 x, u32 n) {
    for (u32 i = 0; i < n; i++) {
        u32 bl = (u32)w[T_BLEN];
        if (bl == 64) {                                      // more input after a full block
            u32 cv[8], m[16]; t_get(w + T_CV, cv);
#pragma unroll
            for (int k = 0; k < 8; k++) put(m, k, w[T_BLOCK + k]);
            const u32 nb = (u32)w[T_NBLK];
            if (nb == 15) {                                  // ... and a full chunk: push its chaining value, merging completed subtrees
                compress_ctr(cv, m, w[T_CTR], 64, CHUNK_END);
                u64 total = w[T_CTR] + 1; u32 sl = (u32)w[T_SLEN];
                while ((total & 1) == 0) {
                    u32 l[8]; t_get(w + T_STACK + 4 * (sl - 1), l);
#pragma unroll
                    for (int k = 0; k < 8; k++) { m[k] = l[k]; m[8 + k] = cv[k]; }
                    iv(cv); compress_ctr(cv, m, 0ULL, 64, PARENT);
                    sl--; total >>= 1;
                }
                if (sl < T_STACK_MAX) { t_put(w + T_STACK + 4 * sl, cv); w[T_SLEN] = (w[T_SLEN] & T_OVERFLOW) | (sl + 1); }
                else w[T_SLEN] = T_OVERFLOW | sl;
                w[T_CTR] += 1; iv(cv); w[T_NBLK] = 0;
            } else {
                compress_ctr(cv, m, w[T_CTR], 64, nb == 0 ? CHUNK_START : 0u);
                w[T_NBLK] = nb + 1;
            }
            t_put(w + T_CV, cv);
#pragma unroll
            for (int k = 0; k < 8; k++) w[T_BLOCK + k] = 0;
            bl = 0;
        }
        reinterpret_cast<unsigned char *>(w + T_BLOCK)[bl] = (unsigned char)(x >> (8 * i));
        w[T_BLEN] = bl + 1;
    }
}
// finalize_xof's first 16 bytes as two little-endian words, non-destructively: the chunk's output, merged with the stack right to
// left, then one ROOT compression at output counter 0
static __device__ __noinline__ void t_finalize16(const u64 *w, u64 &a, u64 &b) {
    u32 cv[8], m[16]; t_get(w + T_CV, cv);
#pragma unroll
    for (int k = 0; k < 8; k++) put(m, k, w[T_BLOCK + k]);
    u64 ctr = w[T_CTR]; u32 len = (u32)w[T_BLEN], flags = (w[T_NBLK] == 0 ? CHUNK_START : 0u) | CHUNK_END;
    for (int i = (int)(u32)w[T_SLEN] - 1; i >= 0; i--) {
        compress_ctr(cv, m, ctr, len, flags);
        u32 l[8]; t_get(w + T_STACK + 4 * i, l);
#pragma unroll
        for (int k = 0; k < 8; k++) { m[k] = l[k]; m[8 + k] = cv[k]; }
        iv(cv); ctr = 0; len = 64; flags = PARENT;
    }
    compress_ctr(cv, m, ctr, len, flags | ROOT);
    a = (u64)cv[0] | ((u64)cv[1] << 32); b = (u64)cv[2] | ((u64)cv[3] << 32);
}

// BlakeTranscript's framing (transcript/src/blake.rs through trait Transcript, host twin: host/transcript.hpp BlakeTranscript)
__host__ __device__ constexpr u64 le_word(const char *s, int n) { u64 v = 0; for (int i = n - 1; i >= 0; i--) v = (v << 8) | (unsigned char)s[i]; return v; }
// the canonical value's little-endian bytes without trailing zeros (BigUint::to_bytes_le: one byte for zero)
__device__ __forceinline__ u32 t_fe_len(u64 c) { return c ? (u32)(71 - __clzll((long long)c)) / 8 : 1u; }
__device__ __forceinline__ void t_append_fe(u64 *w, u64 f) {                  // "field_element" + bytes(f)
    const u64 c = gl_canon(f);
    t_absorb(w, le_word("field_el", 8), 8); t_absorb(w, le_word("ement", 5), 5); t_absorb(w, c, t_fe_len(c));
}
__device__ __forceinline__ void t_append_ext(u64 *w, u64 c0, u64 c1) {        // "field_element_ext" + bytes(c0) + bytes(c1)
    c0 = gl_canon(c0); c1 = gl_canon(c1);
    t_absorb(w, le_word("field_el", 8), 8); t_absorb(w, le_word("ement_ex", 8), 8); t_absorb(w, le_word("t", 1), 1);
    t_absorb(w, c0, t_fe_len(c0)); t_absorb(w, c1, t_fe_len(c1));
}
// read_challenge: "challenge", 16 output bytes as two words, again while either is not canonical
__device__ __forceinline__ void t_challenge(u64 *w, u64 &a, u64 &b) {
    do { t_absorb(w, le_word("challeng", 8), 8); t_absorb(w, le_word("e", 1), 1); t_finalize16(w, a, b); } while (a >= GL_P || b >= GL_P);
}
}  // namespace b3

// TrB3: BlakeTranscript as a transcript policy of the resident sumcheck kernels (see TrP2 in poseidon2.cuh), the hasher above on
// thread 0, working on the image in place.
struct TrB3 {
    static constexpr int WORDS = b3::T_STACK + 4 * b3::T_STACK_MAX;
    __device__ static bool runs() { return threadIdx.x == 0; }
    u64 *w;
    __device__ explicit TrB3(u64 *img) : w(img) {}
    __device__ void ext(gle e) { b3::t_append_ext(w, e.c0, e.c1); }
    __device__ void usize(u64 v) { b3::t_append_fe(w, v); }
    __device__ void label(const u64 (&l)[2]) { b3::t_append_fe(w, l[0]); b3::t_append_fe(w, l[1]); }   // one field element per 8 bytes
    __device__ gle challenge() { u64 a, b; b3::t_challenge(w, a, b); return e_make(a, b); }
    __device__ void store(u64 *dst, u64 *also) { for (int i = 0; i < WORDS; i++) { if (dst != w) dst[i] = w[i]; if (also) also[i] = w[i]; } }
};
