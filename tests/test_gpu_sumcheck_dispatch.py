"""Every sumcheck round-kernel variant against the oracle, round by round.

dp_sc_round picks one of three kernel families per round from the shape of the polynomial at that round (lean k_sc_lean<D, MODE>,
general k_sc_round<DSEL>, resident tail k_sc_res<DSEL>), and each family has further branches inside.  `dispatch` below restates
the host-side routing of deep-prove_b200/csrc/sumcheck.cu in Python; CASES is a matrix of small polynomials (num_vars <= 16) that,
run through the model, reaches every cell in REQUIRED_CELLS.  The CPU test checks that coverage; the GPU tests run each case with
the resident tail off and on and check the messages, the folded tables, the final evaluations and -- through the kernel profile --
that the device took the path the model predicts.  A second set repeats a few cases with adversarial values (tables of p - 1,
alternating 0 / p - 1, challenges 0, 1, p - 1, non-canonical challenges) that drive the lazy 96/160/192-bit sums into their carries.
"""
import ctypes as C
import os
import zlib
from collections import Counter, namedtuple

import numpy as np
import pytest

import oracle_py as O

P = O.P

# ---- constants of sumcheck.cu the model depends on -----------------------------------------------------------------------------
SC_THREADS = 256            # SC_THREADS: threads per block of k_sc_round and k_sc_res
WARP = 32
LEAN_MIN_PAIRS = 2048       # dp_sc_round's lean-kernel choice: lean kernels only when the round has MORE pairs than this
SC_RES_WORK = 2048          # SC_RES_WORK: resident once the round's pair-items, summed over products, are <= this
SC_RES_CTA_WORK = 512       # sc_res_shape: ~pair-items per CTA of the resident cluster
SC_RES_MAXCTA = 8           # SC_RES_MAXCTA
SC_RES_MAXP = 48            # SC_RES_MAXP
SC_RES_MAXM = 96            # SC_RES_MAXM
COUNTER_POOL_BYTES = 256    # dp_sc_create's pooled counters: tick counters (n_products + 1 u32) come from a pooled 256-byte block when they fit
H100_SMS = 132              # common.cuh DpCtx::sm_count default; on the device the real count is read from torch
# sc_tail_supported: the tail disables itself under tools that serialise launches
INJECTION_VARS = ("CUDA_INJECTION64_PATH", "CUDA_INJECTION32_PATH", "NV_NSIGHT_INJECTION_TRANSPORT_TYPE",
                  "NV_NSIGHT_INJECTION_PORT_BASE", "NV_COMPUTE_PROFILER_PERFWORKS_DIR")

LEAN_PROFILE_NAME = {"B": "k_sc_lean(msg, Base)", "E": "k_sc_lean(msg, Ext)", "BF": "k_sc_lean(fold Base->Ext + msg)",
                     "EF": "k_sc_lean(fold Ext + msg)"}


def _grid_for(work, threads, max_ctas_per_sm, sm_count):          # common.cuh dp_grid_for
    return int(max(1, min((work + threads - 1) // threads, sm_count * max_ctas_per_sm)))


def res_ncta(work):                                                 # :757
    n = 1
    while n < SC_RES_MAXCTA and n * SC_RES_CTA_WORK < work:
        n <<= 1
    return n


def res_groups(n_products, ncta):                                   # :503-505  warps per product, a power of two
    W = ncta * (SC_THREADS // WARP)
    G = 1
    while n_products * (G << 1) <= W:
        G <<= 1
    return W, G


def _dsel(products):                                                # :761-762, :889-890  one degree for all products, else 0
    d = len(products[0])
    return d if all(len(p) == d for p in products) else 0


def dispatch(mle_shapes, products, max_nv, tail, sm_count=H100_SMS):
    """mle_shapes: [(num_vars, 'b' | 'e')]; products: [[mle index]]; tail: dp_sc_set_resident_tail took effect.
    Returns one dict per round describing the kernel dp_sc_round runs for it."""
    lens = [1 << nv for nv, _ in mle_shapes]
    ext = [k == "e" for _, k in mle_shapes]
    n_m, n_p = len(mle_shapes), len(products)
    used = {i for p in products for i in p}
    s_gx = min((max([1] + [ln >> 1 for ln in lens]) + 127) // 128 + 1, sm_count * 16)      # :815-825
    res = None
    rounds = []
    for k in range(max_nv):
        fold = k > 0
        folds = [fold and ln > 1 for ln in lens]                    # :870-879 (and :515 in the kernel)
        if res is None and tail:
            # sc_tail_eligible (:726-730) with sc_round_work (:721-725): the length of each product's FIRST operand decides
            work = sum(max(((lens[p[0]] >> 1) if folds[p[0]] else lens[p[0]]) >> 1, 1) for p in products)
            eligible = (n_m <= SC_RES_MAXM and n_p <= SC_RES_MAXP and max_nv - k >= 2
                        and all(i in used or lens[i] <= 1 for i in range(n_m)) and work <= SC_RES_WORK)
            if eligible:
                ncta = res_ncta(work)
                W, G = res_groups(n_p, ncta)
                res = dict(dsel=_dsel(products), ncta=ncta, W=W, G=G, round0=(k == 0), start=k)
        descs = []                                                  # the descriptors of sc_desc (:460-478), built by dp_sc_round (:884) and the kernel (:520)
        for p in products:
            modes = [("EF" if ext[i] else "BF") if folds[i] else ("E" if ext[i] else "B") for i in p]
            newlen = (lens[p[0]] >> 1) if folds[p[0]] else lens[p[0]]
            descs.append(dict(d=len(p), modes=modes, konst=newlen == 1, npairs=newlen >> 1,
                              allbase=all(m == "B" for m in modes), square=len(set(p)) < len(p)))
        if res is not None:
            prods = []
            for d in descs:
                tpl = 2 if d["d"] <= 3 else 3                       # :550-551
                split = not d["konst"] and not d["allbase"] and (d["npairs"] << tpl) <= res["G"] * WARP
                prods.append(dict(split=split, konst=d["konst"], square=d["square"]))
            rounds.append(dict(family="resident", first=(k == res["start"]), products=prods, **res))
        else:
            dsel = _dsel(products)
            round_pairs = max([1] + [d["npairs"] for d in descs])
            lean = None                                             # :891-899
            if dsel in (2, 3) and round_pairs > LEAN_MIN_PAIRS:
                m0 = descs[0]["modes"][0]
                if all(not d["konst"] and all(m == m0 for m in d["modes"]) for d in descs):
                    lean = m0
            if lean == "B":                                         # :907-910
                gx = min((round_pairs + 511) // 512, sm_count * 4)
            elif lean is not None:
                gx = min((round_pairs + 127) // 128, s_gx)
            elif round_pairs > 8192:
                gx = min(s_gx, _grid_for(round_pairs, SC_THREADS, 6, sm_count))
            else:
                gx = min(s_gx, _grid_for(round_pairs if round_pairs <= 256 else (round_pairs + 1) // 2, SC_THREADS, 4, sm_count))
            transport = "param" if n_p == 1 else ("device" if gx * n_p > 32 else "mapped")       # :922-924
            counters = "pooled" if 4 * (n_p + 1) <= COUNTER_POOL_BYTES else "dedicated"       # :832-833
            r = dict(gx=gx, transport=transport, counters=counters, round_pairs=round_pairs)
            if lean is not None:
                r.update(family="lean", D=dsel, mode=lean, profile=LEAN_PROFILE_NAME[lean],
                         npairs=[d["npairs"] for d in descs])
            else:
                bodies = [dict(body="const" if d["konst"] else ("allbase" if d["allbase"] else "general"), square=d["square"])
                          for d in descs]
                r.update(family="general", dsel=dsel, products=bodies, profile="k_sc_round(fold+msg)" if fold else "k_sc_round(msg)")
            rounds.append(r)
        for i in range(n_m):                                        # commit the folds (sc_commit_fold, :454; :933 and :585)
            if folds[i]:
                lens[i] >>= 1
                ext[i] = True
    return rounds


def expected_profile(plan):
    """launches per k_sc_* profile name: one per per-round kernel, one for the whole resident tail"""
    c = Counter(r["profile"] for r in plan if r["family"] != "resident")
    if any(r["family"] == "resident" for r in plan):
        c["k_sc_res"] = 1
    return dict(c)


# ---- the case matrix ---------------------------------------------------------------------------------------------------------
Case = namedtuple("Case", "name nv mles products")


def uni(name, nv, shape):
    """every product gets its own MLEs of num_vars nv; shape: [[kind per operand]]"""
    mles, products = [], []
    for kinds in shape:
        products.append(list(range(len(mles), len(mles) + len(kinds))))
        mles += [(nv, k) for k in kinds]
    return Case(name, nv, mles, products)


def _edge_48p_96m():
    return Case("res_edge_48p_96m_d2", 4, [(4, "be"[i % 2]) for i in range(96)], [[2 * i, 2 * i + 1] for i in range(48)])


def _edge_49p():
    return Case("noneligible_49p_96m", 4, [(4, "be"[i % 2]) for i in range(96)],
                [[2 * i, 2 * i + 1] for i in range(47)] + [[94], [95]])


def _edge_97m():
    return Case("noneligible_48p_97m", 4, [(4, "be"[i % 2]) for i in range(97)],
                [[2 * i, 2 * i + 1] for i in range(47)] + [[94, 95, 96]])


CASES = [
    # lean: all 8 (D, MODE) cells; Base inputs reach B, BF and EF, Ext inputs E and EF
    uni("lean_B2_BF2_EF2_gen2_res2mid", 15, [["b", "b"]]),
    uni("lean_B3_BF3_EF3_gen3_res3mid", 15, [["b", "b", "b"]]),
    uni("lean_E2_EF2_res2mid", 14, [["e", "e"]]),
    uni("lean_E3_EF3_device_descs", 14, [["e", "e", "e"], ["e", "e", "e"]]),
    # lean with products of different num_vars (the smaller one 2048 pairs in round 0); later a constant product in both paths
    Case("lean_B2_mixed_nv_then_const", 15, [(15, "b"), (15, "b"), (12, "b"), (12, "b")], [[0, 1], [2, 3]]),
    # general kernels, each DSEL with gridDim.x > 1, and the resident tail of each DSEL from round 0 / mid-proof
    uni("gen1_allbase_res1_round0_G32", 12, [["b"]]),
    uni("gen1_res1_mid_G32", 13, [["e"]]),
    uni("gen2_res2_round0_G16", 11, [["e", "b"], ["b", "e"]]),
    uni("gen3_allbase_res3_round0", 12, [["b", "b", "b"]]),
    uni("gen4_res4_round0", 12, [["e", "b", "b", "e"]]),
    uni("gen4_res4_mid", 13, [["b", "e", "b", "b"]]),
    uni("gen5_res5_round0", 12, [["b", "e", "b", "e", "b"]]),
    uni("gen5_res5_mid", 13, [["e", "e", "b", "b", "b"]]),
    uni("gen0_mapped_descs_res0_mid", 12, [["b", "b", "b", "b", "b"], ["e", "e", "e", "e"]]),
    uni("res0_round0_G8", 10, [["e", "b"], ["e", "e", "e"], ["b"]]),
    # 64 products: tick counters outside the pooled block, descriptors through a device copy
    Case("gen2_64_products", 10, [(10, "be"[i % 2]) for i in range(16)], [[p % 16, (5 * p + 3) % 16] for p in range(64)]),
    # resident: more products than warps (one warp serves several slots), plain then split bodies
    uni("res_more_products_than_warps", 6, [["e", "b"]] * 12),
    # constant products (smaller num_vars) and a squared MLE, in the general kernel (tail off) and in the tail
    Case("mixed_sizes_const_square", 8, [(8, "e"), (8, "b"), (8, "e"), (3, "b"), (3, "e")],
         [[0, 1, 2], [0, 1], [3, 4], [0, 2, 2], [3]]),
    # an MLE shared by three products whose first reference is operand 1 (and one whose first reference is operand 2)
    Case("res_shared_mle_not_first_operand_ncta2", 9, [(9, "e"), (9, "b"), (9, "e"), (9, "b")], [[1, 0], [0, 2, 3], [3, 0]]),
    # eligibility edges: 48 products / 96 MLEs are resident, 49 products or 97 MLEs are not
    _edge_48p_96m(),
    _edge_49p(),
    _edge_97m(),
]
CASE_BY_NAME = {c.name: c for c in CASES}


def _shared_not_first_operand(case):
    first, count = {}, Counter()
    for p in case.products:
        for j, i in enumerate(p):
            first.setdefault(i, j)
        for i in set(p):
            count[i] += 1
    return any(count[i] >= 2 and first[i] != 0 for i in first)


def cells_of(case, tail):
    """the dispatch cells a case reaches (tail: whether the resident tail is enabled)"""
    plan = dispatch(case.mles, case.products, case.nv, tail)
    cells = set()
    n_p, n_m = len(case.products), len(case.mles)
    for k, r in enumerate(plan):
        if r["family"] == "lean":
            cells.add(("lean", r["D"], r["mode"]))
            if len(set(r["npairs"])) > 1 and min(r["npairs"]) > 1:
                cells.add(("lean", "mixed num_vars"))
        elif r["family"] == "general":
            cells.add(("general", r["dsel"]))
            if r["gx"] > 1:
                cells.add(("general", r["dsel"], "gridDim.x > 1"))
            for b in r["products"]:
                cells.add(("general body", b["body"]))
                if b["square"]:
                    cells.add(("general body", "squared MLE"))
        if r["family"] != "resident":
            cells.add(("descriptors", r["transport"]))
            cells.add(("counters", r["counters"]))
        else:
            if r["first"]:
                cells.add(("resident", r["dsel"], "round 0" if r["round0"] else "mid-proof"))
                cells.add(("resident ncta", r["ncta"]))
                cells.add(("resident gather", "per warp (G >= 32)" if r["G"] >= 32 else "per thread (G < 32)"))
                if n_p > r["W"]:
                    cells.add(("resident", "more products than warps"))
                if _shared_not_first_operand(case):
                    cells.add(("resident", "shared MLE first referenced by operand > 0"))
                if n_p == SC_RES_MAXP and n_m == SC_RES_MAXM:
                    cells.add(("resident", "48 products / 96 MLEs"))
            for p in r["products"]:
                cells.add(("resident body", "split" if p["split"] else "plain"))
                if p["konst"]:
                    cells.add(("resident body", "constant product"))
                if p["square"]:
                    cells.add(("resident body", "squared MLE"))
    if tail and not any(r["family"] == "resident" for r in plan):
        if n_p == SC_RES_MAXP + 1:
            cells.add(("not resident", "49 products"))
        if n_m == SC_RES_MAXM + 1 and len({i for p in case.products for i in p}) == n_m:
            cells.add(("not resident", "97 MLEs, all referenced"))
    return cells


REQUIRED_CELLS = (
    {("lean", d, m) for d in (2, 3) for m in ("B", "E", "BF", "EF")} | {("lean", "mixed num_vars")}
    | {("general", d) for d in range(6)} | {("general", d, "gridDim.x > 1") for d in range(6)}
    | {("general body", b) for b in ("allbase", "const", "general", "squared MLE")}
    | {("descriptors", t) for t in ("param", "mapped", "device")} | {("counters", "pooled"), ("counters", "dedicated")}
    | {("resident", d, w) for d in range(6) for w in ("round 0", "mid-proof")}
    | {("resident ncta", n) for n in (1, 2, 4)}
    | {("resident gather", "per warp (G >= 32)"), ("resident gather", "per thread (G < 32)")}
    | {("resident", "more products than warps"), ("resident", "shared MLE first referenced by operand > 0"),
       ("resident", "48 products / 96 MLEs")}
    | {("resident body", b) for b in ("split", "plain", "constant product", "squared MLE")}
    | {("not resident", "49 products"), ("not resident", "97 MLEs, all referenced")}
)


def test_case_matrix_reaches_every_dispatch_cell():
    covered = set()
    for case in CASES:
        assert case.nv <= 16, case.name
        covered |= cells_of(case, False) | cells_of(case, True)
    missing = REQUIRED_CELLS - covered
    assert not missing, "no case reaches: %s" % sorted(missing, key=str)


def test_resident_cluster_never_needs_8_ctas():
    """~512 pair-items per CTA below SC_RES_WORK = 2048 gives clusters of 1, 2 or 4 CTAs; if the threshold grows, the 8-CTA
    cluster becomes reachable and needs a case of its own in CASES (and a cell in REQUIRED_CELLS)"""
    assert {res_ncta(w) for w in range(1, SC_RES_WORK + 1)} == {1, 2, 4}


def test_model_restates_known_routes():
    """spot checks of the model against routes derived by hand from sumcheck.cu"""
    r = dispatch([(12, "b")] * 3, [[0, 1, 2]], 12, False)
    assert r[0]["family"] == "general" and r[0]["dsel"] == 3 and r[0]["gx"] == 4     # exactly 2048 pairs: not lean
    r = dispatch([(13, "b")] * 3, [[0, 1, 2]], 13, True)
    assert (r[0]["family"], r[0]["mode"]) == ("lean", "B") and r[1]["family"] == "resident" and r[1]["ncta"] == 4
    assert r[1]["G"] == 32 and not r[1]["round0"]
    r = dispatch([(6, "e")] * 2, [[0, 1]], 6, True)
    assert r[0]["family"] == "resident" and r[0]["ncta"] == 1 and r[-1]["family"] == "resident"
    r = dispatch([(1, "b")], [[0]], 1, True)                                          # a single round is never resident
    assert r[0]["family"] == "general"


# ---- inputs -----------------------------------------------------------------------------------------------------------------
def _seed(name):
    return zlib.crc32(name.encode()) & 0xFFFFFF


def make_inputs(case, pattern="random"):
    """(mles, products) in the oracle's format: mles [(array, is_ext)], products [((c0, c1), [idx])]"""
    s = _seed(case.name)
    mles = []
    for i, (nv, kind) in enumerate(case.mles):
        n, is_ext = 1 << nv, kind == "e"
        if pattern == "random":
            a = O.splitmix_e(s + 7 * i, n) if is_ext else O.splitmix_f(s + 7 * i, n)
        else:
            v = np.full(n, P - 1, dtype=np.uint64)
            if pattern == "alternating":
                v[0::2] = 0
            a = np.repeat(v[:, None], 2, axis=1) if is_ext else v
        mles.append((np.ascontiguousarray(a), is_ext))
    if pattern == "random":
        coefs = [tuple(int(x) for x in O.splitmix_e(s + 1000 + p, 1)[0]) for p in range(len(case.products))]
    else:
        coefs = [(P - 1, P - 1)] * len(case.products)
    return mles, [(c, list(p)) for c, p in zip(coefs, case.products)]


EDGE_CHALLENGES = [(0, 0), (1, 0), (P - 1, 0), (P - 1, P - 1), (0, P - 1)]


def edge_challenges(n, seed):
    rng = np.random.default_rng(seed)
    return np.array([EDGE_CHALLENGES[i] for i in rng.integers(0, len(EDGE_CHALLENGES), n)], dtype=np.uint64)


def non_canonical(ch):
    """every limb below 2^32 - 1 as limb + p (still a u64); the library must reduce it to the same element"""
    out = ch.copy()
    small = out < np.uint64(2**32 - 1)
    out[small] += np.uint64(P)
    return out


def test_fold_expectation_for_smaller_mles_matches_the_oracle():
    """The folded-table check of the GPU tests expects MLE i after k rounds to be fix_low(f_i, ch[:min(k, nv_i)]): an MLE with
    fewer variables stops folding once it is a single value.  Confirm that against the oracle's final evaluations, which are
    what a fully folded table must end as."""
    for name in ("lean_B2_mixed_nv_then_const", "mixed_sizes_const_square", "res_shared_mle_not_first_operand_ncta2",
                 "res_edge_48p_96m_d2"):
        case = CASE_BY_NAME[name]
        mles, products = make_inputs(case)
        ch = O.splitmix_e(_seed(name) + 5, case.nv)
        _, fin = O.sumcheck_rounds_fixed(mles, products, case.nv, ch)
        for i, ((a, ext), (nv, _)) in enumerate(zip(mles, case.mles)):
            assert (O.fix_low(a, ext, ch[:nv])[0] == fin[i]).all(), (name, i)


# ---- device runs ------------------------------------------------------------------------------------------------------------
def _tail_supported():
    return not any(v in os.environ for v in INJECTION_VARS)


@pytest.fixture
def kernel_profile(gpu):
    """the profile table is process-wide: enable and clear it for one test only"""
    gpu.profile_enable(True)
    gpu.profile_reset()
    try:
        yield
    finally:
        gpu.profile_enable(False)
        gpu.profile_reset()


@pytest.fixture(scope="module")
def sm_count(gpu):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def current_table(gpu, sc, i):
    h = C.c_void_p()
    gpu.check(gpu.lib().dp_sc_current_mle(sc.h, i, C.byref(h)))
    return gpu.Mle(h.value).download()                  # non-owning view: freeing it leaves the table alone


def run_case(gpu, case, mles, products, ch, tail, sm_count, check_tables=True, sent=None):
    """all rounds of `case` on the device (challenges `sent`, default `ch`) against the oracle with challenges `ch`;
    returns the model's plan"""
    exp_msgs, exp_fin = O.sumcheck_rounds_fixed(mles, products, case.nv, ch)
    plan = dispatch(case.mles, case.products, case.nv, tail and _tail_supported(), sm_count)
    sent = ch if sent is None else sent
    dm = [gpu.Mle.upload(a, e) for a, e in mles]
    sc = gpu.Sumcheck(dm, products, case.nv, max(len(p) for p in case.products))
    try:
        gpu.check(gpu.lib().dp_sc_set_resident_tail(sc.h, int(tail)))
        for k in range(case.nv):
            got = sc.round(None if k == 0 else sent[k - 1])
            what = "%s tail=%d round %d %s" % (case.name, tail, k, {x: y for x, y in plan[k].items() if x != "products"})
            assert (got == exp_msgs[k]).all(), what
            if plan[k]["family"] == "resident":
                with pytest.raises(gpu.DpError) as e:
                    current_table(gpu, sc, 0)
                assert e.value.code == gpu.DP_ERR_STATE, what
            elif check_tables:
                for i, ((a, ext), (nv, _)) in enumerate(zip(mles, case.mles)):
                    t = current_table(gpu, sc, i)
                    exp = a if k == 0 else O.fix_low(a, ext, ch[:min(k, nv)])
                    assert t.shape == exp.shape and (t == exp).all(), "%s: MLE %d" % (what, i)
        assert (sc.finish(sent[case.nv - 1]) == exp_fin).all(), "%s tail=%d final evaluations" % (case.name, tail)
    finally:
        sc.destroy()
    for m, (a, _) in zip(dm, mles):
        assert (m.download() == a).all(), "%s tail=%d: an input MLE was modified" % (case.name, tail)
    return plan


def check_profile(gpu, case, tail, plan):
    got = {}
    for name, (count, _, _) in gpu.profile_read().items():
        if name.startswith("k_sc_res"):           # the name is cut to 63 characters
            name = "k_sc_res"
        if name.startswith("k_sc_"):
            got[name] = got.get(name, 0) + count
    assert got == expected_profile(plan), "%s tail=%d: launches per kernel differ from the dispatch model" % (case.name, tail)


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [0, 1], ids=["tail_off", "tail_on"])
@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_dispatch_case(gpu, kernel_profile, sm_count, name, tail):
    """every round message, every folded table (tail off), the final evaluations and the untouched inputs against the oracle;
    the launches per kernel name against the model's route"""
    case = CASE_BY_NAME[name]
    mles, products = make_inputs(case)
    ch = O.splitmix_e(_seed(name) + 5, case.nv)
    plan = run_case(gpu, case, mles, products, ch, bool(tail), sm_count)
    check_profile(gpu, case, tail, plan)


VALUE_EDGE_CASES = ["lean_B2_BF2_EF2_gen2_res2mid",       # lean B, BF, EF
                    "lean_E3_EF3_device_descs",           # lean E, EF
                    "gen0_mapped_descs_res0_mid",         # general, mixed degrees
                    "gen3_allbase_res3_round0",           # resident: plain body, then split from round 3
                    "res_more_products_than_warps"]       # resident: several slots per warp, split body


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [0, 1], ids=["tail_off", "tail_on"])
@pytest.mark.parametrize("pattern", ["all_p_minus_1", "alternating_0_p_minus_1"])
@pytest.mark.parametrize("name", VALUE_EDGE_CASES)
def test_dispatch_value_edges(gpu, sm_count, name, pattern, tail):
    """tables (and coefficients) at p - 1 or alternating 0 / p - 1, challenges from {0, 1, p - 1, (p - 1, p - 1), (0, p - 1)}:
    the largest limbs the lazy sums can see; the same challenges again with every limb below 2^32 - 1 sent as limb + p"""
    case = CASE_BY_NAME[name]
    mles, products = make_inputs(case, "alternating" if pattern.startswith("alternating") else "max")
    ch = edge_challenges(case.nv, _seed(name + pattern))
    plan = run_case(gpu, case, mles, products, ch, bool(tail), sm_count, check_tables=False)
    if tail and _tail_supported():
        assert any(r["family"] == "resident" for r in plan)
    sent = non_canonical(ch)
    assert (sent != ch).any()
    run_case(gpu, case, mles, products, ch, bool(tail), sm_count, check_tables=False, sent=sent)


def _extrapolate(vals, x):
    """Lagrange interpolation over the points 0..len(vals)-1, evaluated at x (per limb: the weights are base-field elements)"""
    n = len(vals)
    out = [0, 0]
    for j in range(n):
        num = den = 1
        for i in range(n):
            if i != j:
                num = num * (x - i) % P
                den = den * (j - i) % P
        w = num * pow(den, P - 2, P) % P
        out = [(out[0] + int(vals[j][0]) * w) % P, (out[1] + int(vals[j][1]) * w) % P]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [0, 1], ids=["tail_off", "tail_on"])
@pytest.mark.parametrize("max_deg", [4, 5])
def test_max_degree_above_product_degree(gpu, max_deg, tail):
    """degree-2 products with a larger max_degree: points 0..2 are the oracle's message, the rest its extrapolation"""
    case = uni("max_degree_d2_B2_then_general_then_resident", 13, [["b", "b"], ["b", "b"]])
    mles, products = make_inputs(case)
    ch = O.splitmix_e(_seed(case.name), case.nv)
    exp_msgs, exp_fin = O.sumcheck_rounds_fixed(mles, products, case.nv, ch)
    sc = gpu.Sumcheck([gpu.Mle.upload(a, e) for a, e in mles], products, case.nv, max_deg)
    try:
        gpu.check(gpu.lib().dp_sc_set_resident_tail(sc.h, tail))
        for k in range(case.nv):
            got = sc.round(None if k == 0 else ch[k - 1])
            assert got.shape == (max_deg + 1, 2)
            assert (got[:3] == exp_msgs[k]).all(), "round %d" % k
            for x in range(3, max_deg + 1):
                assert [int(v) for v in got[x]] == _extrapolate(exp_msgs[k], x), "round %d point %d" % (k, x)
        assert (sc.finish(ch[-1]) == exp_fin).all()
    finally:
        sc.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("max_deg", [6, 7, 16])
def test_max_degree_above_5_is_rejected(gpu, max_deg):
    """the round message holds at most 6 points (prover.rs:710: "do not support degree > 5")"""
    a = gpu.Mle.upload(O.splitmix_f(1, 16), False)
    b = gpu.Mle.upload(O.splitmix_f(2, 16), False)
    with pytest.raises(gpu.DpError) as e:
        gpu.Sumcheck([a, b], [((1, 0), [0, 1])], 4, max_deg)
    assert e.value.code == gpu.DP_ERR_UNSUPPORTED and "do not support degree > 5" in str(e.value)
