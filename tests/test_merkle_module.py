"""CPU tests: the Merkle trees live in one module.  csrc/merkle.cu holds every tree kernel, the tree layout (LvlOff, QTree), the
hasher switch and its copy of the Poseidon2 constants; basefold.cu reaches them only through merkle.cuh, includes neither hash
header, and a tree owns what it stores (no ownership flags, views or separate level-0 buffers beside it)."""
import re

from test_launch_rule import sources

# names that belong to merkle.cu alone (poseidon2.cuh defines p2_upload_constants, and only merkle.cu may call it)
MODULE_ONLY = [r"\bk_merkle_\w+", r"\bk_b3_\w+", r"\bk_leafpair_root\b", r"\bk_query_gather\b", r"\bLvlOff\b", r"\bQTree\b",
               r"\bp2_upload_constants\b", r"\bg_hasher\b", r"\bdp_set_merkle_hasher\b", r"\bdp_get_merkle_hasher\b"]
GONE = ["own_levels", "own_level0", "tree_view", "top_lvl0", "rt_done"]


def test_tree_code_lives_in_merkle_cu():
    srcs = sources()
    assert "merkle.cu" in srcs and "merkle.cuh" in srcs
    for pat in MODULE_ONLY:
        assert re.search(pat, srcs["merkle.cu"]), "merkle.cu lacks " + pat
        exempt = ("merkle.cu", "poseidon2.cuh") if pat == r"\bp2_upload_constants\b" else ("merkle.cu",)
        where = sorted(name for name, src in srcs.items() if name not in exempt and re.search(pat, src))
        assert where == [], "%s outside merkle.cu: %s" % (pat, where)


def test_basefold_includes_no_hash_header():
    includes = re.findall(r'#include\s+"([^"]+)"', sources()["basefold.cu"])
    assert "merkle.cuh" in includes
    assert not {"poseidon2.cuh", "blake3.cuh"} & set(includes), includes


def test_trees_own_what_they_store():
    for name, src in sources().items():
        for word in GONE:
            assert word not in src, "%s still uses %s" % (name, word)
