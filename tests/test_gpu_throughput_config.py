"""The configuration the benchmark measures -- many proofs in flight, proving threads asleep on the library's poller
(dp_set_wait_mode(1)) -- against the oracle.

Several device paths exist only in that configuration:
  * the Merkle builder changes shape with the wait mode (deep-prove_b200/csrc/merkle.cu tree_build, :233-306): in block mode
    k_merkle_small takes 256-hash subtrees, hashes every level of >= 64 hashes one thread per hash (p2_compress_lat) and folds
    up to 8 subtree roots in the last block; in spin mode it takes 32-hash subtrees, always uses the 8-lane p2x8_compress and
    folds up to 64.  `tree_plan` below restates tree_build rule by rule; CASES is a matrix of commitments that, run through the
    model, reaches every cell in REQUIRED_CELLS in both modes.  The GPU tests check the root, the codeword, the evaluations and
    (nv > 7) the whole opening proof against the oracle, and -- through the kernel profile -- that the device built the tree
    the way the model says;
  * every host wait goes through a one-thread signal kernel and the poller instead of cudaStreamSynchronize (csrc/context.cu
    dp_stream_sync), so a root, a D2H result or a round message reaches the host only through stream order and that kernel's
    system fence.  The Basefold, resident sumcheck tail and zkml parity checks run again in block mode;
  * dp_pcs_commit_many spreads commitments over 4 streams in block mode (8 in spin mode) and recycles stream sets between host
    threads;
  * the concurrent prover pool (host/capi.cpp): per-worker contexts, staggered starts from a pool's second call, the shared
    Merkle ticket ring.  dph_zkml_prove_concurrent_all returns every job's proof, and each must equal the oracle's.

The ticket ring (merkle.cu:150-163, :280, MK_TICKETS = 4096 counters handed out round robin) is safe only while fewer than 4096
k_merkle_small launches lie between one launch's enqueue and its completion.  A proof commits about 38 witness trees per
dp_pcs_commit_many call (basefold.cu:556) and its thread waits for the call to finish, so 48 proofs in flight hold at most
about 48 x 38 = 1.8 k launches: a margin of about 2x.  Nothing here tries to provoke a collision.
"""
import ctypes as C
import threading
import zlib
from collections import Counter, namedtuple

import numpy as np
import pytest

import dpb200
import models
import oracle_py as O
import test_gpu_basefold as B
import test_gpu_sumcheck_dispatch as S
import test_zkml as Z

P = O.P
SPIN, BLOCK = 0, 1

# ---- constants of merkle.cu the model depends on ------------------------------------------------------------------------------
MK_SMALL = 2048             # :81   k_merkle_small builds every remaining level once a level has <= this many hashes
MK_SUB = 256                # :80   hashes of the first level per block in block mode
SPIN_SUB = 32               # :278  ... and in spin mode
TPH_MIN = 64                # :278  block mode: a block level with >= this many hashes runs one thread per hash
MK_MID_MAX = 32768          # :287  k_merkle_mid up to this many hashes per level, k_merkle_wide above
B3_TAIL_MAX = 1024          # :269  BLAKE3: k_b3_tail takes every remaining level once a level has <= this many hashes
BF_BASECODE_LOG = 7         # nv <= 7: a trivial commitment, the tree is over the evaluations themselves
BF_RATE_LOG = 1             # otherwise the tree is over the 2^(nv + 1) codeword entries

PROFILE_NAME = {            # DpProfScope names of tree_build's kernels (k_leafpair_root has none)
    "k_merkle_small": "k_merkle_small(poseidon2 compress, all remaining levels)",
    "k_merkle_mid": "k_merkle_mid(poseidon2 compress, thread per hash)",
    "k_merkle_wide": "k_merkle(poseidon2 compress)",
    "k_leafpair_root": None,
    "k_b3_leaves": "k_b3_leaves(blake3)",
    "k_b3_up": "k_b3_up(blake3)",
    "k_b3_tail": "k_b3_tail(blake3)",
}
TREE_PROFILE_NAMES = {v for v in PROFILE_NAME.values() if v}


def tree_plan(n_leaves, ext, batch_lvl0, hasher, wait_mode):
    """tree_build (merkle.cu:233-306) for a tree over n_leaves leaves.  batch_lvl0: the leaf-pair digests are given (a batch
    commitment); hasher: "poseidon2" or "blake3".  Returns dict(lg, launches: Counter of kernel names, route: [(kernel, level,
    hashes, source)], small: None or the k_merkle_small launch as dict(first_level, hashes, source, ext, grid, sub,
    levels: [(hashes per block, "thread" | "8 lanes")], fold: [hashes per fold level]))."""
    lg = 0
    while (1 << lg) < n_leaves:                                                    # :235
        lg += 1
    assert lg >= 1                                                                 # :236
    launches, route, small = Counter(), [], None
    if hasher == "blake3":                                                         # :268-273
        if not batch_lvl0:                                                         # :241-254  level 0 is stored
            launches["k_b3_leaves"] += 1
        for l in range(1, lg):                                                     # :263
            nl = n_leaves >> (l + 1)
            if nl <= B3_TAIL_MAX:                                                  # :269
                launches["k_b3_tail"] += 1
                route.append(("k_b3_tail", l, nl, None))
                break
            launches["k_b3_up"] += 1                                               # :270-271
            route.append(("k_b3_up", l, nl, None))
        return dict(lg=lg, launches=launches, route=route, small=None)
    if lg == 1:                                                                    # :258-262
        if not batch_lvl0:
            launches["k_leafpair_root"] += 1
            route.append(("k_leafpair_root", 0, 1, "leaves"))
        return dict(lg=lg, launches=launches, route=route, small=None)
    for l in range(1, lg):                                                         # :263
        nl = n_leaves >> (l + 1)
        source = ("batch level 0" if batch_lvl0 else "leaves") if l == 1 else "digests"     # :265-266
        if nl <= MK_SMALL:                                                         # :275
            many = wait_mode == BLOCK                                              # :277-278
            sub_max, tph_min = (MK_SUB, TPH_MIN) if many else (SPIN_SUB, None)
            grid = (nl + sub_max - 1) // sub_max                                   # :279
            sub = min(nl, sub_max)                                                 # kernel :93
            levels, lv, k = [], l, 0
            while (sub >> k) >= 1 and lv < lg:                                     # kernel :95-125
                cnt = sub >> k
                levels.append((cnt, "thread" if tph_min is not None and cnt >= tph_min else "8 lanes"))
                k += 1
                lv += 1
            fold = []
            if grid > 1:                                                           # kernel :126, :134-146
                cnt = grid >> 1
                while cnt >= 1 and lv < lg:
                    fold.append(cnt)
                    cnt >>= 1
                    lv += 1
            assert lv == lg, "k_merkle_small must end at the root"
            small = dict(first_level=l, hashes=nl, source=source, ext=ext and source == "leaves", grid=grid, sub=sub,
                         levels=levels, fold=fold)
            launches["k_merkle_small"] += 1
            route.append(("k_merkle_small", l, nl, source))
            break
        kernel = "k_merkle_mid" if nl <= MK_MID_MAX else "k_merkle_wide"         # :287, :301
        launches[kernel] += 1
        route.append((kernel, l, nl, source))
    return dict(lg=lg, launches=launches, route=route, small=small)


def expected_profile(plan):
    """launches per profile name of tree_build's kernels"""
    c = Counter()
    for k, n in plan["launches"].items():
        if PROFILE_NAME[k]:
            c[PROFILE_NAME[k]] += n
    return dict(c)


# ---- the case matrix ---------------------------------------------------------------------------------------------------------
Case = namedtuple("Case", "name hasher nv ext n_polys full_log")   # n_polys > 1: one batch commitment (Basefold::batch_commit)


def n_leaves(case):
    return 1 << case.nv if case.nv <= BF_BASECODE_LOG else 1 << (case.nv + BF_RATE_LOG)


def plan_of(case, wait_mode):
    return tree_plan(n_leaves(case), case.ext, case.n_polys > 1, case.hasher, wait_mode)


CASES = [
    # Poseidon2, one polynomial
    Case("p2_lg1_nv1_base", "poseidon2", 1, False, 1, 8),                # k_leafpair_root
    Case("p2_trivial_nv3_ext", "poseidon2", 3, True, 1, 8),              # small from Ext leaves, grid 1
    Case("p2_trivial_nv7_base", "poseidon2", 7, False, 1, 9),            # small from Base leaves, grid 1, 8 lanes only
    Case("p2_nv8_base", "poseidon2", 8, False, 1, 8),                    # block: grid 1, threads at 128, 64; spin: grid 4
    Case("p2_nv9_ext", "poseidon2", 9, True, 1, 11),                     # block: grid 1, threads from Ext leaves; spin: grid 8
    Case("p2_nv10_base", "poseidon2", 10, False, 1, 10),                 # block: fold over 2
    Case("p2_nv11_ext", "poseidon2", 11, True, 1, 12),                   # block: fold over 4, Ext leaves
    Case("p2_nv12_base", "poseidon2", 12, False, 1, 14),                 # block: fold over 8; spin: fold over 64
    Case("p2_nv12_ext", "poseidon2", 12, True, 1, 12),                   # the same from Ext leaves
    Case("p2_nv13_base", "poseidon2", 13, False, 1, 13),                 # mid from Base leaves, then small from digests
    Case("p2_nv14_ext", "poseidon2", 14, True, 1, 15),                   # mid from Ext leaves, mid from digests
    Case("p2_nv16_base", "poseidon2", 16, False, 1, 16),                 # four mid levels, then small from digests
    Case("p2_nv17_base", "poseidon2", 17, False, 1, 17),                 # k_merkle_wide from Base leaves
    Case("p2_nv17_ext", "poseidon2", 17, True, 1, 17),                   # k_merkle_wide from Ext leaves
    Case("p2_nv18_base", "poseidon2", 18, False, 1, 19),                 # k_merkle_wide from leaves, then from digests
    # Poseidon2, batch commitments (the leaf-pair digests of all polynomials are level 0)
    Case("p2_batch_lg1_nv1", "poseidon2", 1, False, 2, 8),               # the root is the level-0 digest
    Case("p2_batch_nv9_base", "poseidon2", 9, False, 3, 10),             # small from level 0 (block: threads, grid 1)
    Case("p2_batch_nv10_ext", "poseidon2", 10, True, 2, 10),             # small from level 0, grid > 1 in both modes
    Case("p2_batch_nv13_base", "poseidon2", 13, False, 3, 13),           # mid from level 0
    Case("p2_batch_nv17_base", "poseidon2", 17, False, 2, 17),           # k_merkle_wide from level 0
    # BLAKE3
    Case("b3_lg1_nv1_base", "blake3", 1, False, 1, 8),
    Case("b3_nv10_ext", "blake3", 10, True, 1, 10),                      # tail only
    Case("b3_nv12_base", "blake3", 12, False, 1, 13),                    # k_b3_up, then the tail
    Case("b3_batch_nv9_base", "blake3", 9, False, 3, 9),                 # from a batch level 0
]
CASE_BY_NAME = {c.name: c for c in CASES}


def cells_of(case, wait_mode):
    """the tree_build cells a case reaches in one wait mode"""
    plan = plan_of(case, wait_mode)
    batch = case.n_polys > 1
    field = "Ext" if case.ext else "Base"
    cells = set()
    if case.hasher == "blake3":
        if plan["lg"] == 1:
            cells.add(("blake3", "lg == 1"))
        kernels = [r[0] for r in plan["route"]]
        if kernels == ["k_b3_tail"]:
            cells.add(("blake3", "tail only"))
        if "k_b3_up" in kernels and kernels[-1] == "k_b3_tail":
            cells.add(("blake3", "k_b3_up then tail"))
        if batch:
            cells.add(("blake3", "batch level 0"))
        return cells
    if plan["lg"] == 1:
        cells.add(("poseidon2", "lg == 1", "batch" if batch else "single"))
    for kernel, _, _, source in plan["route"]:
        if kernel == "k_merkle_mid":
            cells.add(("k_merkle_mid", source, field) if source == "leaves" else ("k_merkle_mid", source))
        elif kernel == "k_merkle_wide":
            cells.add(("k_merkle_wide", source, field) if source == "leaves" else ("k_merkle_wide", source))
    s = plan["small"]
    if s is not None:
        grid = "grid 1" if s["grid"] == 1 else "grid > 1"
        cells.add(("k_merkle_small", s["source"], field, grid) if s["source"] == "leaves" else ("k_merkle_small", s["source"]))
        for _, branch in s["levels"]:
            if branch == "thread":
                cells.add(("k_merkle_small", "thread per hash", "leaves" if s["source"] == "leaves" else "digests"))
            else:
                cells.add(("k_merkle_small", "8 lanes"))
        if s["fold"]:
            cells.add(("k_merkle_small", "fold over", s["grid"]))
    return cells


COMMON_CELLS = (
    {("poseidon2", "lg == 1", w) for w in ("single", "batch")}
    | {("k_merkle_small", "leaves", f, g) for f in ("Base", "Ext") for g in ("grid 1", "grid > 1")}
    | {("k_merkle_small", "digests"), ("k_merkle_small", "batch level 0"), ("k_merkle_small", "8 lanes")}
    | {("k_merkle_mid", "leaves", f) for f in ("Base", "Ext")} | {("k_merkle_mid", "digests"), ("k_merkle_mid", "batch level 0")}
    | {("k_merkle_wide", "leaves", f) for f in ("Base", "Ext")} | {("k_merkle_wide", "digests"), ("k_merkle_wide", "batch level 0")}
    | {("blake3", c) for c in ("lg == 1", "tail only", "k_b3_up then tail", "batch level 0")}
)
REQUIRED_CELLS = {
    SPIN: COMMON_CELLS | {("k_merkle_small", "fold over", 64)},
    BLOCK: COMMON_CELLS | {("k_merkle_small", "thread per hash", s) for s in ("leaves", "digests")}
    | {("k_merkle_small", "fold over", g) for g in (2, 4, 8)},
}


@pytest.fixture(scope="module", autouse=True)
def _module_leaves_spin_mode():
    yield
    assert dpb200.lib().dp_get_wait_mode() == SPIN, "a test left the process in blocking wait mode"


@pytest.mark.parametrize("wait_mode", [SPIN, BLOCK], ids=["spin", "block"])
def test_case_matrix_reaches_every_tree_cell(wait_mode):
    covered = set()
    for case in CASES:
        covered |= cells_of(case, wait_mode)
    missing = REQUIRED_CELLS[wait_mode] - covered
    assert not missing, "no case reaches: %s" % sorted(missing, key=str)


def test_model_restates_known_routes():
    """routes derived by hand from merkle.cu"""
    # nv = 12 (Base): 2^13 leaves, level 1 has 2048 hashes -> k_merkle_small from the leaves
    r = tree_plan(1 << 13, False, False, "poseidon2", BLOCK)
    s = r["small"]
    assert dict(r["launches"]) == {"k_merkle_small": 1} and s["first_level"] == 1 and s["hashes"] == 2048
    assert s["grid"] == 8 and s["levels"] == [(256, "thread"), (128, "thread"), (64, "thread")] + [(c, "8 lanes") for c in (32, 16, 8, 4, 2, 1)]
    assert s["fold"] == [4, 2, 1]
    r = tree_plan(1 << 13, False, False, "poseidon2", SPIN)
    s = r["small"]
    assert s["grid"] == 64 and [b for _, b in s["levels"]] == ["8 lanes"] * 6 and len(s["fold"]) == 6
    # nv = 16: four k_merkle_mid levels, then k_merkle_small from digests
    for mode in (SPIN, BLOCK):
        r = tree_plan(1 << 17, False, False, "poseidon2", mode)
        assert [k for k, *_ in r["route"]] == ["k_merkle_mid"] * 4 + ["k_merkle_small"]
        assert r["small"]["source"] == "digests" and r["small"]["hashes"] == 2048
    # nv = 17 starts with k_merkle_wide, then k_merkle_mid (32768 hashes is still a mid level)
    r = tree_plan(1 << 18, True, False, "poseidon2", BLOCK)
    assert r["route"][0][:3] == ("k_merkle_wide", 1, 1 << 16) and r["route"][1][:3] == ("k_merkle_mid", 2, 1 << 15)
    # a tree of two leaves: no launch from a batch level 0, k_leafpair_root otherwise; BLAKE3 stores its level 0
    assert not tree_plan(2, False, True, "poseidon2", BLOCK)["launches"]
    assert dict(tree_plan(2, False, False, "poseidon2", SPIN)["launches"]) == {"k_leafpair_root": 1}
    assert dict(tree_plan(1 << 13, False, False, "blake3", SPIN)["launches"]) == {"k_b3_leaves": 1, "k_b3_up": 1, "k_b3_tail": 1}
    # every level from 1 up to the root is built exactly once, in both modes
    for n in range(2, 21):
        for mode in (SPIN, BLOCK):
            r = tree_plan(1 << n, False, False, "poseidon2", mode)
            s = r["small"]
            per_launch = [lv for _, lv, _, _ in r["route"]]
            top = s["first_level"] + len(s["levels"]) + len(s["fold"]) if s else r["lg"]
            assert per_launch == list(range(1, len(per_launch) + 1)) and top == r["lg"], (n, mode)


# ---- device runs ------------------------------------------------------------------------------------------------------------
def _set_mode(gpu, mode):
    before = gpu.lib().dp_get_wait_mode()
    gpu.set_wait_mode(mode)
    return before


@pytest.fixture(params=[SPIN, BLOCK], ids=["spin", "block"])
def wait_mode(gpu, request):
    """runs the test in spin and in blocking wait mode; restores the previous mode"""
    before = _set_mode(gpu, request.param)
    try:
        yield request.param
    finally:
        gpu.set_wait_mode(before)


@pytest.fixture
def block_mode(gpu):
    before = _set_mode(gpu, BLOCK)
    try:
        yield BLOCK
    finally:
        gpu.set_wait_mode(before)


@pytest.fixture
def hasher(gpu, request):
    """the case's Merkle hasher on the device and in the oracle (process-wide switches), Poseidon2 again afterwards"""
    kind = 1 if request.param == "blake3" else 0
    O.set_hash_mode(kind)
    gpu.set_hasher(kind)
    try:
        yield request.param
    finally:
        O.set_hash_mode(0)
        gpu.set_hasher(0)


def _injected_tools():
    return not S._tail_supported()       # a profiler or sanitizer injected into the CUDA runtime


def _seed(name):
    return zlib.crc32(name.encode()) & 0xFFFFFF


def make_polys(case, pattern="random"):
    """the case's polynomials: random, or value edges of the first permutation (all 0, all p - 1 -- (p - 1, p - 1) for Ext --,
    alternating 0 / p - 1)"""
    s, n = _seed(case.name), 1 << case.nv
    polys = []
    for i in range(case.n_polys):
        if pattern == "random":
            a = O.splitmix_e(s + 11 * i, n) if case.ext else O.splitmix_f(s + 11 * i, n)
        else:
            v = np.full(n, 0 if pattern == "zeros" else P - 1, dtype=np.uint64)
            if pattern == "alternating":
                v[(i & 1)::2] = 0
            a = np.repeat(v[:, None], 2, axis=1) if case.ext else v
        polys.append(np.ascontiguousarray(a))
    return polys


def _root(gpu, h):
    root = np.zeros(4, dtype=np.uint64)
    gpu.check(gpu.lib().dp_pcs_comm_info(h, None, None, None, root.ctypes.data_as(C.c_void_p)))
    return root


def _comm_data(gpu, h):
    """(root, bit-reversed codeword, bit-reversed evaluations) of a dp_pcs_comm handle of one polynomial"""
    root = _root(gpu, h)
    v = C.c_void_p()
    gpu.check(gpu.lib().dp_pcs_comm_codeword(h, C.byref(v)))
    cw = gpu.Mle(v.value).download()                     # non-owning views
    gpu.check(gpu.lib().dp_pcs_comm_bh_evals(h, C.byref(v)))
    return root, cw, gpu.Mle(v.value).download()


def commit_on_device(gpu, case, polys):
    """one dp_pcs_commit (or dp_pcs_batch_commit) -> (root, [(codeword, evaluations) per polynomial])"""
    L = gpu.lib()
    mles = [gpu.Mle.upload(p, case.ext) for p in polys]
    h = C.c_void_p()
    if case.n_polys == 1:
        gpu.check(L.dp_pcs_commit(mles[0].h, case.full_log, C.byref(h)))
    else:
        gpu.check(L.dp_pcs_batch_commit(gpu.handles(mles), len(mles), case.full_log, C.byref(h)))
    try:
        if case.n_polys == 1:
            root, cw, bh = _comm_data(gpu, h)
            return root, [(cw, bh)]
        root, parts = _root(gpu, h), []      # a batch commitment: the codewords belong to its per-polynomial views
        for i in range(case.n_polys):
            ph = C.c_void_p()
            gpu.check(L.dp_pcs_comm_part(h, i, C.byref(ph)))
            parts.append(_comm_data(gpu, ph)[1:])
        return root, parts
    finally:
        L.dp_pcs_comm_free(h)


def check_commit(gpu, case, polys, wait_mode, check_profile=True):
    """root, codewords and evaluations against the oracle; the Merkle launches against the model"""
    profile = check_profile and not _injected_tools()
    if profile:
        gpu.profile_enable(True)
        gpu.profile_reset()
    try:
        root, parts = commit_on_device(gpu, case, polys)
        got_profile = {k: v[0] for k, v in gpu.profile_read().items() if k in TREE_PROFILE_NAMES} if profile else None
    finally:
        if profile:
            gpu.profile_enable(False)
            gpu.profile_reset()
    what = "%s mode=%d" % (case.name, wait_mode)
    for i, (p, (cw, bh)) in enumerate(zip(polys, parts)):
        _, ecw, ebh = O.pcs_commit(p, case.ext, case.full_log)
        assert bh.shape == ebh.shape and (bh == ebh).all(), "%s: evaluations of polynomial %d" % (what, i)
        assert cw.shape == ecw.shape and (cw == ecw).all(), "%s: codeword of polynomial %d" % (what, i)
    if case.n_polys == 1:
        eroot = O.pcs_commit(polys[0], case.ext, case.full_log, want_codeword=False)[0]
    else:
        eroot = O.pcs_simple_batch(polys, case.ext, case.full_log)[0]
    assert (root == eroot).all(), "%s: root" % what
    if profile:
        plan = plan_of(case, wait_mode)
        assert got_profile == expected_profile(plan), "%s: Merkle launches per kernel differ from the model %s" % (what, plan["route"])


def check_open(gpu, case, polys, wait_mode):
    """the whole opening proof word for word (its query paths read every stored level back; its own oracle trees are small)"""
    what = "%s mode=%d" % (case.name, wait_mode)
    pt = O.splitmix_e(_seed(case.name) + 1, case.nv)
    mles = [gpu.Mle.upload(p, case.ext) for p in polys]
    if case.n_polys == 1:
        exp = O.pcs_open(polys[0], case.ext, case.full_log, pt)
        _, got = gpu.pcs_open(mles[0], case.full_log, pt)
    else:
        _, evals, exp = O.pcs_simple_batch(polys, case.ext, case.full_log, pt)
        _, got = gpu.pcs_simple_batch(mles, case.full_log, pt, evals)
    if got.shape != exp.shape or not (got == exp).all():
        n = min(got.size, exp.size)
        bad = np.nonzero(got[:n] != exp[:n])[0]
        raise AssertionError("%s: opening proof differs: %d vs %d words, first difference at word %s"
                             % (what, got.size, exp.size, bad[0] if bad.size else n))


@pytest.mark.gpu
@pytest.mark.parametrize("name,hasher", [(c.name, c.hasher) for c in CASES], indirect=["hasher"])
def test_tree_case(gpu, wait_mode, hasher, name):
    case = CASE_BY_NAME[name]
    polys = make_polys(case)
    check_commit(gpu, case, polys, wait_mode)
    if case.nv > BF_BASECODE_LOG:
        check_open(gpu, case, polys, wait_mode)


VALUE_EDGE_CASES = ["p2_trivial_nv7_base",     # 8 lanes straight from the polynomial's values
                    "p2_trivial_nv3_ext",      # ... Ext values
                    "p2_nv9_ext",              # block: thread per hash from Ext leaves
                    "p2_nv12_base",            # block: threads, 8 lanes and the fold over 8; spin: fold over 64
                    "p2_nv13_base",            # k_merkle_mid from leaves, small from digests
                    "p2_nv17_ext",             # k_merkle_wide from Ext leaves
                    "p2_batch_nv9_base"]       # a batch level 0


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["zeros", "all_p_minus_1", "alternating"])
@pytest.mark.parametrize("name", VALUE_EDGE_CASES)
def test_tree_value_edges(gpu, wait_mode, name, pattern):
    case = CASE_BY_NAME[name]
    polys = make_polys(case, pattern)
    check_commit(gpu, case, polys, wait_mode, check_profile=False)
    if case.nv > BF_BASECODE_LOG:
        check_open(gpu, case, polys, wait_mode)


# ---- dp_pcs_commit_many, called directly ---------------------------------------------------------------------------------------
# 19 polynomials (more than the 8 streams of spin mode and the 4 of block mode): trivial ones (nv <= 7), k_encode_small sizes
# (the codeword fits in 64 KiB), tiled-path sizes (nv 13-16, Ext 12+), Base and Ext interleaved
MANY_SHAPES = [(3, False), (5, True), (7, False), (8, False), (9, True), (10, False), (11, True), (12, False), (13, False), (13, True),
               (14, False), (15, True), (16, False), (6, True), (9, False), (12, True), (10, True), (14, True), (8, True)]
MANY_FULL_LOG = 16


def _many_polys(seed):
    return [(O.splitmix_e(seed + i, 1 << nv) if ext else O.splitmix_f(seed + i, 1 << nv), ext) for i, (nv, ext) in enumerate(MANY_SHAPES)]


def commit_many_on_device(gpu, polys):
    """one dp_pcs_commit_many call -> [(root, codeword, evaluations)]"""
    L = gpu.lib()
    mles = [gpu.Mle.upload(a, e) for a, e in polys]
    out = (C.c_void_p * len(mles))()
    gpu.check(L.dp_pcs_commit_many(gpu.handles(mles), len(mles), MANY_FULL_LOG, out))
    try:
        return [_comm_data(gpu, out[i]) for i in range(len(mles))]
    finally:
        for i in range(len(mles)):
            L.dp_pcs_comm_free(out[i])


def check_many(gpu, polys, got, what):
    for i, ((a, ext), (root, cw, bh)) in enumerate(zip(polys, got)):
        eroot, ecw, ebh = O.pcs_commit(a, ext, MANY_FULL_LOG)
        assert (root == eroot).all(), "%s: root of commitment %d" % (what, i)
        assert cw.shape == ecw.shape and (cw == ecw).all(), "%s: codeword of commitment %d" % (what, i)
        assert bh.shape == ebh.shape and (bh == ebh).all(), "%s: evaluations of commitment %d" % (what, i)


def _in_new_thread(gpu, fn):
    """fn() on a fresh host thread with its own library context (and, when one is free, a recycled set of commit streams)"""
    box = {}

    def run():
        try:
            gpu.init(0)
            try:
                box["value"] = fn()
            finally:
                gpu.lib().dp_shutdown()
        except BaseException as e:      # re-raised on the calling thread
            box["error"] = e

    t = threading.Thread(target=run)
    t.start()
    t.join()
    if "error" in box:
        raise box["error"]
    return box["value"]


@pytest.mark.gpu
def test_commit_many(gpu, wait_mode):
    """each commitment of one call equals the oracle's and a single dp_pcs_commit of the same polynomial; a second call on the
    same thread reuses its stream set, calls from new threads take a recycled one"""
    polys = _many_polys(7000)
    what = "commit_many mode=%d" % wait_mode
    got = commit_many_on_device(gpu, polys)
    check_many(gpu, polys, got, what)
    for i, ((a, ext), (root, cw, bh)) in enumerate(zip(polys, got)):
        c = gpu.Commitment(gpu.Mle.upload(a, ext), MANY_FULL_LOG)
        assert (c.root == root).all() and (c.codeword() == cw).all() and (c.bh_evals() == bh).all(), "%s: commitment %d vs dp_pcs_commit" % (what, i)
        c.free()
    polys2 = _many_polys(7100)
    check_many(gpu, polys2, commit_many_on_device(gpu, polys2), what + ", second call")
    # the first new thread returns its stream set when it exits, the second one takes it
    check_many(gpu, polys2, _in_new_thread(gpu, lambda: commit_many_on_device(gpu, polys2)), what + ", new thread")
    check_many(gpu, polys, _in_new_thread(gpu, lambda: commit_many_on_device(gpu, polys)), what + ", thread with a recycled stream set")


# ---- every proof of a concurrent call -----------------------------------------------------------------------------------------
def _first_difference(proofs, exp):
    """(job, word) of the first proof that differs from `exp`, or None"""
    for j, got in enumerate(proofs):
        if got.size != exp.size or not (got == exp).all():
            n = min(got.size, exp.size)
            bad = np.nonzero(got[:n] != exp[:n])[0]
            return j, int(bad[0]) if bad.size else n
    return None


def check_concurrent(ctx, exp, n_workers, n_proofs, e2e, what, calls=2):
    """`calls` calls of n_proofs jobs on n_workers workers (from a pool's second call the workers start staggered): every job's
    proof equals the oracle's"""
    for call in range(calls):
        _, proofs, workers = ctx.prove_concurrent_all(n_workers, n_proofs, stride=exp.size + 64, e2e=e2e)
        assert len(proofs) == n_proofs and (workers < n_workers).all(), what
        bad = _first_difference(proofs, exp)
        if bad is not None:
            j, w = bad
            raise AssertionError("%s, call %d: job %d (worker %d, %d words against %d) first differs at word %d"
                                 % (what, call, j, workers[j], proofs[j].size, exp.size, w))


_SMALL_MODELS = {}


def small_model(gpu, name):
    """(context with a stored trace, oracle proof), built once per module"""
    if name not in _SMALL_MODELS:
        if name == "mlp_2x128":
            w, b, rq = O.synthetic_mlp(2, 128, 21)
            x = O.synthetic_input(128, 22)
            ctx = gpu.ZkmlContext(2, 128, w, b, rq)
            exp, _ = O.zkml_prove(2, 128, 21, 22)
        else:
            desc, data, x, _ = models.cnn_small(seed=5)
            ctx = gpu.ModelContext(desc, data, x.size)
            exp, _ = O.model_prove(desc, data, x)
        ctx.run_inference(x)
        _SMALL_MODELS[name] = (ctx, exp)
    return _SMALL_MODELS[name]


@pytest.fixture(scope="module")
def small_models(gpu):
    yield lambda name: small_model(gpu, name)
    for ctx, _ in _SMALL_MODELS.values():
        ctx.free()                       # joins the pool's worker threads
    _SMALL_MODELS.clear()


@pytest.mark.gpu
@pytest.mark.parametrize("e2e", [False, True], ids=["resident", "e2e"])
@pytest.mark.parametrize("n_workers", [1, 4, 16])
@pytest.mark.parametrize("model", ["mlp_2x128", "cnn_small"])
def test_concurrent_small_models(gpu, small_models, wait_mode, model, n_workers, e2e):
    ctx, exp = small_models(model)
    check_concurrent(ctx, exp, n_workers, 3 * n_workers, e2e, "%s workers=%d e2e=%d mode=%d" % (model, n_workers, e2e, wait_mode))


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["dense4m", "cnn264k"])
def test_concurrent_benchmark_configurations(gpu, block_mode, model):
    """the benchmark's configurations: 48 workers, 96 proofs, blocking waits, resident and end to end; one oracle proof
    serves every job"""
    if model == "dense4m":
        w, b, rq = O.synthetic_mlp(4, 1024, 1)
        x = O.synthetic_input(1024, 2)
        ctx = gpu.ZkmlContext(4, 1024, w, b, rq)
        exp, _ = O.zkml_prove(4, 1024, 1, 2)
    else:
        desc, data, x, _ = models.cnn(seed=7)
        ctx = gpu.ModelContext(desc, data, x.size)
        exp, _ = O.model_prove(desc, data, x)
    try:
        ctx.run_inference(x)
        for e2e in (False, True):
            check_concurrent(ctx, exp, 48, 96, e2e, "%s e2e=%d" % (model, e2e), calls=1)
    finally:
        ctx.free()


# ---- existing parity checks again with blocking waits ---------------------------------------------------------------------
def _params(fn):
    """the parameter sets of a parametrized test function"""
    return [m.args[1] for m in fn.pytestmark if m.name == "parametrize"][0]


@pytest.mark.gpu
@pytest.mark.parametrize("nv,full_log,ext", _params(B.test_commit))
def test_basefold_commit_block_mode(gpu, block_mode, nv, full_log, ext):
    B.test_commit(gpu, nv, full_log, ext)


@pytest.mark.gpu
@pytest.mark.parametrize("nv,full_log,ext", _params(B.test_open))
def test_basefold_open_block_mode(gpu, block_mode, nv, full_log, ext):
    B.test_open(gpu, nv, full_log, ext)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,full_log", _params(B.test_batch_open))
def test_basefold_batch_open_block_mode(gpu, block_mode, shape, full_log):
    B.test_batch_open(gpu, shape, full_log)


@pytest.mark.gpu
@pytest.mark.parametrize("n_polys,nv,full_log,ext", _params(B.test_batch_commit_and_simple_batch_open))
def test_basefold_simple_batch_block_mode(gpu, block_mode, n_polys, nv, full_log, ext):
    B.test_batch_commit_and_simple_batch_open(gpu, n_polys, nv, full_log, ext)


RESIDENT_TAIL_CASES = [c.name for c in S.CASES if any(r["family"] == "resident" for r in S.dispatch(c.mles, c.products, c.nv, True))]


def test_resident_tail_cases_exist():
    assert len(RESIDENT_TAIL_CASES) >= 10


@pytest.mark.gpu
@pytest.mark.parametrize("name", RESIDENT_TAIL_CASES)
def test_sumcheck_resident_tail_block_mode(gpu, block_mode, name):
    """the resident tail's round messages reach the host through the poller in block mode"""
    import torch
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    case = S.CASE_BY_NAME[name]
    mles, products = S.make_inputs(case)
    ch = O.splitmix_e(S._seed(name) + 5, case.nv)
    gpu.profile_enable(True)
    gpu.profile_reset()
    try:
        plan = S.run_case(gpu, case, mles, products, ch, True, sm_count)
        S.check_profile(gpu, case, 1, plan)
    finally:
        gpu.profile_enable(False)
        gpu.profile_reset()


@pytest.mark.gpu
@pytest.mark.parametrize("nl,width", _params(Z.test_proof_parity))
def test_zkml_proof_parity_block_mode(gpu, block_mode, nl, width):
    """the LogUp outputs reach the host through mapped memory and the poller in block mode"""
    Z.test_proof_parity(gpu, nl, width)
