// The Merkle trees of the Basefold PCS and their query paths (merkle.cu).  Host-side declarations only.
#pragma once
#include "common.cuh"

// batch trees: at most MK_BATCH_MAX leaf vectors, and under BLAKE3 at most MK_B3_BATCH_WORDS words of values at one index
static constexpr u32 MK_BATCH_MAX = 64;
static constexpr u32 MK_B3_BATCH_WORDS = 128;
bool mk_blake3();   // the process-wide hasher (dp_set_merkle_hasher) is BLAKE3 rather than Poseidon2

// A tree over 2^lg leaves.  The leaves are not part of it: they are a commitment's codeword or a round's oracle, passed in to
// build the tree and to query it.  Level 0, one digest per leaf pair, is stored for BLAKE3 trees, batch trees and sharded top
// trees (whose level 0 is the G subtree roots); a single-polynomial Poseidon2 tree recomputes it from the leaves, since it is the
// zero-padded pair itself (hash_or_noop of <= 4 elements).  Levels 1 .. lg-1 are packed back to back.  The tree owns both.
struct DevTree {
    u32 lg = 0; bool ext = false;
    u64 *level0 = nullptr;
    u64 *levels = nullptr;
    const u64 *root_dev = nullptr;   // 4 words in level0 or levels
    bool root_published = false;     // the build's last launch also handed the root over through its RootOut
};
// hand-over of the root by the launch that computes it: root words into mapped pinned memory, a system fence, then `seq` in `flag`
struct RootOut { u64 *root_host; u64 *flag; u64 seq; };

// `leaves`: one vector, or up to MK_BATCH_MAX for a batch tree (Basefold::batch_commit).  `rt` may be null.
int tree_build(DevTree &t, const std::vector<const void *> &leaves, bool ext, u64 n, const RootOut *rt = nullptr);
int top_tree_build(DevTree &top, const uint64_t *roots, u32 logG, uint64_t root[4]);   // roots: 4 words per rank, rank-major
void tree_free(DevTree &t);

// One tree a query opens: its leaves, the shift from the query index to theirs, and the sharded top tree.  mk_query_words gives a
// query's row length in u64 words (and each tree's offset in it); mk_query_gather writes the rows.
struct MkPath { const DevTree *tree; const void *leaves; u32 shift; const DevTree *top; };
u64 mk_query_words(const std::vector<MkPath> &paths, u32 logG, std::vector<u64> *row_off = nullptr);
int mk_query_gather(const std::vector<MkPath> &paths, u32 logG, u32 rank, const uint64_t *x_indices, u32 n, uint64_t *out);
