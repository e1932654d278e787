"""The device side of the lookup argument against a big-integer reference, cell by cell and at value edges.

LogUp-GKR circuit (deep-prove_b200/csrc/logup.cu): dp_logup_build computes the denominators in k_logup_den, streams the large
layers through k_logup_layer and finishes every small one in the single-block k_logup_tail; the first layer of a lookup circuit
(numerators all -1) is done by k_logup_layer<true> or by the tail's lookup branch, depending on its size.  `logup_plan` restates
that routing; LOGUP_CASES reaches every {lookup, table} x {tail only, one streamed layer, several streamed layers} cell.  Each case
checks every layer's views, the outputs, the untouched inputs and -- through the kernel profile -- the launches the plan predicts,
against `ref_circuit`, a restatement of circuit.rs in Python integers.  The helpers the LogUp prover calls
(dp_mle_linear_combination, dp_mle_evaluate_many) and the lookup-witness kernels (csrc/witness.cu: dense, matmul, requant, relu,
maxpool, multiplicities) are checked the same way, at the table ends and at the error boundaries.
"""
import ctypes as C
import zlib
from collections import namedtuple

import numpy as np
import pytest

import oracle_py as O
from test_gpu_witness import to_field

P = O.P
SPIN, BLOCK = 0, 1
EDGE_CHALLENGES = [(0, 0), (1, 0), (P - 1, 0), (P - 1, P - 1), (0, P - 1)]


def _seed(name):
    return zlib.crc32(name.encode()) & 0xFFFFFF


# ---- reference: LogUpCircuit in Python integers (zkml/src/lookup/logup_gkr/circuit.rs) --------------------------------------
def _obj(a):
    return np.array([int(v) for v in np.asarray(a, dtype=np.uint64).reshape(-1)], dtype=object)


def _ext_obj(a):
    a = np.asarray(a, dtype=np.uint64).reshape(-1, 2)
    return _obj(a[:, 0]), _obj(a[:, 1])


def _ext_u64(v):
    return np.stack([v[0].astype(np.uint64), v[1].astype(np.uint64)], axis=1)


def _canon(e):
    return int(e[0]) % P, int(e[1]) % P


def _vmul(a, b):
    """(a0 + a1 X)(b0 + b1 X) with X^2 = 7, elementwise"""
    return (a[0] * b[0] + 7 * a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P


def _vadd(a, b):
    return (a[0] + b[0]) % P, (a[1] + b[1]) % P


def ref_denominators(cols, c, gamma):
    """c + sum_k gamma^k col_k[i]  (circuit.rs:207-224 for lookups, :242-262 for tables)"""
    c, gamma = _canon(c), _canon(gamma)
    n = len(cols[0])
    d = (np.full(n, c[0], dtype=object), np.full(n, c[1], dtype=object))
    pw = (1, 0)
    for col in cols:
        v = _obj(col)
        d = _vadd(d, ((pw[0] * v) % P, (pw[1] * v) % P))
        pw = O.pe_mul(pw, gamma)
    return d


def ref_next_layer(num, den):
    """(n1 d2 + d1 n2, d1 d2), pairing i with i + half (circuit.rs:66-80, structs.rs Fraction add); num None: the initial lookup
    layer, whose numerators are all -1 (circuit.rs:82-98)"""
    h = len(den[0]) // 2
    d1, d2 = (den[0][:h], den[1][:h]), (den[0][h:], den[1][h:])
    if num is None:
        s = _vadd(d1, d2)
        n = ((-s[0]) % P, (-s[1]) % P)
    else:
        n = _vadd(_vmul((num[0][:h], num[1][:h]), d2), _vmul(d1, (num[0][h:], num[1][h:])))
    return n, _vmul(d1, d2)


def ref_circuit(cols, mult, c, gamma):
    """every layer, bottom to top, as [(num (n, 2) u64 or None, den (n, 2) u64)]: LogUpCircuit::new (circuit.rs:192-196) from
    new_lookup_circuit (mult None) or new_table_circuit (numerators = the multiplicities lifted to E, :249-252); the last layer
    has 2 fractions (num_vars 0, circuit.rs:43-53)"""
    den = ref_denominators(cols, c, gamma)
    num = None if mult is None else (_obj(mult), np.zeros(len(mult), dtype=object))
    layers = [(num, den)]
    while len(den[0]) > 2:
        num, den = ref_next_layer(num, den)
        layers.append((num, den))
    return [(None if n is None else _ext_u64(n), _ext_u64(d)) for n, d in layers]


def ref_outputs(layers):
    """LogUpCircuit::outputs (circuit.rs:273-275): flat_evals of the last layer, [n0, n1, d0, d1]"""
    n, d = layers[-1]
    return np.concatenate([n, d])


# ---- routing model of dp_logup_build (logup.cu) --------------------------------------------------------------------------
STREAM_MIN_HALF = 1024      # logup.cu:110  a layer is streamed while its output (half) has MORE than this many fractions


def logup_plan(nv, table):
    """nv = log2 of the column length.  logup.cu:107 one k_logup_den; :109-117 k_logup_layer for layer k while
    k + 1 < nv and len >> (k + 1) > 1024 (k = 0 with a lookup circuit is the <true> variant); :118-125 one k_logup_tail from
    the first layer not streamed, whose lookup branch (:48) serves layer 0 only when the tail starts there"""
    k = 0
    while k + 1 < nv and (1 << (nv - k - 1)) > STREAM_MIN_HALF:
        k += 1
    return dict(streamed=k, tail_from=k, tail=k + 1 < nv,
                first_lookup=None if table else ("k_logup_layer<true>" if k > 0 else "k_logup_tail"))


def expected_profile(nv, table):
    plan = logup_plan(nv, table)
    exp = {"k_logup_den": 1, "k_logup_tail": int(plan["tail"])}
    if plan["streamed"]:
        exp["k_logup_layer"] = plan["streamed"]
    return exp


def plan_cell(nv, table):
    s = logup_plan(nv, table)["streamed"]
    return ("table" if table else "lookup", "tail only" if s == 0 else ("one streamed layer" if s == 1 else "several streamed layers"))


# ---- the case matrix ---------------------------------------------------------------------------------------------------------
LCase = namedtuple("LCase", "name nv ncols table cols ch mult")


def _shape_cases():
    out = []
    for table, shapes in ((False, [(2, 1), (3, 2), (11, 3), (12, 16), (13, 2), (14, 3)]),
                          (True, [(2, 3), (3, 16), (11, 1), (12, 16), (13, 3), (14, 2)])):
        for nv, nc in shapes:
            kind = "table" if table else "lookup"
            out.append(LCase("%s_nv%d_%dcols" % (kind, nv, nc), nv, nc, table, "random", "random", "random" if table else None))
    return out


def _edge_cases():
    out = []
    for nv in (3, 12):                      # the first lookup layer in the tail / in k_logup_layer<true>
        for table in (False, True):
            kind = "table" if table else "lookup"
            m = "random" if table else None
            for ch in ("zero", "one", "p_minus_1", "non_canonical", "gamma_zero"):
                out.append(LCase("%s_nv%d_ch_%s" % (kind, nv, ch), nv, 3, table, "random", ch, m))
            out.append(LCase("%s_nv%d_cols_p_minus_1" % (kind, nv), nv, 3, table, "p_minus_1", "p_minus_1", m))
            out.append(LCase("%s_nv%d_cols_alternating" % (kind, nv), nv, 3, table, "alternating", "p_minus_1", m))
            out.append(LCase("%s_nv%d_cols_zero_c_zero" % (kind, nv), nv, 3, table, "zero", "c_zero", m))
            if table:
                out.append(LCase("table_nv%d_mult_zero" % nv, nv, 2, True, "random", "random", "zero"))
                out.append(LCase("table_nv%d_mult_p_minus_1" % nv, nv, 2, True, "p_minus_1", "p_minus_1", "p_minus_1"))
    return out


LOGUP_CASES = _shape_cases() + _edge_cases()
LOGUP_BY_NAME = {c.name: c for c in LOGUP_CASES}
REQUIRED_CELLS = {(k, r) for k in ("lookup", "table") for r in ("tail only", "one streamed layer", "several streamed layers")}


def _column(pattern, n, seed, k):
    if pattern == "random":
        return O.splitmix_f(seed, n)
    if pattern == "zero":
        return np.zeros(n, dtype=np.uint64)
    v = np.full(n, P - 1, dtype=np.uint64)
    if pattern == "alternating":
        v[k % 2::2] = 0
    return v


def _challenges(pattern, seed):
    """(c, gamma) the reference uses, (c, gamma) sent to the library"""
    r = O.splitmix_e(seed, 2)
    c, g = {"random": (r[0], r[1]), "zero": ((0, 0), (0, 0)), "one": ((1, 0), (1, 0)),
            "p_minus_1": ((P - 1, P - 1), (P - 1, P - 1)), "gamma_zero": (r[0], (0, 0)), "c_zero": ((0, 0), r[1]),
            "non_canonical": (r[0] & np.uint64(0x7FFFFFFF), r[1] & np.uint64(0x7FFFFFFF))}[pattern]
    c, g = np.array(c, dtype=np.uint64), np.array(g, dtype=np.uint64)
    if pattern == "non_canonical":            # every limb is below 2^31: sent as limb + p, still a u64
        return (c, g), (c + np.uint64(P), g + np.uint64(P))
    return (c, g), (c, g)


def make_logup_inputs(case):
    s = _seed(case.name)
    n = 1 << case.nv
    cols = [_column(case.cols, n, s + 11 * k, k) for k in range(case.ncols)]
    mult = None
    if case.table:
        mult = {"random": lambda: O.splitmix_f(s + 500, n), "zero": lambda: np.zeros(n, dtype=np.uint64),
                "p_minus_1": lambda: np.full(n, P - 1, dtype=np.uint64)}[case.mult]()
    ref_ch, sent_ch = _challenges(case.ch, s + 1000)
    return cols, mult, ref_ch, sent_ch


def test_case_matrix_reaches_every_routing_cell():
    covered = {plan_cell(c.nv, c.table) for c in LOGUP_CASES}
    missing = REQUIRED_CELLS - covered
    assert not missing, "no case reaches: %s" % sorted(missing)
    assert {c.nv for c in LOGUP_CASES} >= {2, 3, 11, 12, 13, 14} and {c.ncols for c in LOGUP_CASES} >= {1, 2, 3, 16}
    assert any(c.ncols == 16 and c.nv >= 12 for c in LOGUP_CASES)
    # the rare value branches: every edge pattern reaches both places the first lookup layer can be computed
    for ch in ("zero", "one", "p_minus_1", "non_canonical", "gamma_zero"):
        assert {logup_plan(c.nv, c.table)["first_lookup"] for c in LOGUP_CASES if c.ch == ch and not c.table} == \
            {"k_logup_tail", "k_logup_layer<true>"}, ch


def test_logup_plan_restates_known_routes():
    """routes derived by hand from logup.cu:106-125"""
    for nv in range(2, 25):
        p = logup_plan(nv, False)
        assert p["streamed"] == max(0, nv - 11) and p["tail"] and p["tail_from"] == p["streamed"]
    assert logup_plan(11, False)["first_lookup"] == "k_logup_tail"          # half = 1024: not streamed
    assert logup_plan(12, False)["first_lookup"] == "k_logup_layer<true>"   # half = 2048
    assert logup_plan(12, True)["first_lookup"] is None
    assert expected_profile(14, True) == {"k_logup_den": 1, "k_logup_layer": 3, "k_logup_tail": 1}
    assert expected_profile(2, False) == {"k_logup_den": 1, "k_logup_tail": 1}


def test_reference_by_hand_4_entries():
    """circuit.rs by hand: one column [0, 1, 2, 3], c = 5, gamma = 1"""
    col = np.arange(4, dtype=np.uint64)
    L = ref_circuit([col], None, (5, 0), (1, 0))
    assert L[0][0] is None and [int(v) for v in L[0][1][:, 0]] == [5, 6, 7, 8]
    # -1/5 + -1/7 = -12/35, -1/6 + -1/8 = -14/48
    assert [[int(x) for x in r] for r in ref_outputs(L)] == [[P - 12, 0], [P - 14, 0], [35, 0], [48, 0]]
    # table: multiplicities [1, 2, 3, 4], two columns [0, 1, 2, 3] and [1, 1, 1, 1], c = 0, gamma = X (the extension generator)
    L = ref_circuit([col, np.ones(4, dtype=np.uint64)], np.array([1, 2, 3, 4], dtype=np.uint64), (0, 0), (0, 1))
    assert [tuple(int(x) for x in r) for r in L[0][1]] == [(0, 1), (1, 1), (2, 1), (3, 1)]
    # 1/(0+X) + 3/(2+X) = (2+X + 3X)/((X)(2+X)) = (2 + 4X)/(7 + 2X);  2/(1+X) + 4/(3+X) = (6+2X + 4+4X)/(3+X+3X+7) = (10 + 6X)/(10 + 4X)
    assert [tuple(int(x) for x in r) for r in ref_outputs(L)] == [(2, 4), (10, 6), (7, 2), (10, 4)]


def oracle_circuit(cols, mult, c, gamma):
    """the C++ oracle's logup_circuit (oracle/zkml.hpp), every layer"""
    L = O.lib()
    n, nv = len(cols[0]), len(cols[0]).bit_length() - 1
    cs = [O.u64(a) for a in cols]
    arr = (C.c_void_p * len(cs))(*[a.ctypes.data for a in cs])
    m = None if mult is None else O.u64(mult)
    cc, gg = O.u64([int(x) % P for x in c]), O.u64([int(x) % P for x in gamma])
    out = np.zeros(sum(2 * (n >> k) for k in range(nv)) * 2, dtype=np.uint64)
    L.dpo_logup_circuit.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.dpo_logup_circuit(arr, len(cs), n, None if m is None else m.ctypes.data, cc.ctypes.data, gg.ctypes.data, out.ctypes.data)
    layers, o = [], 0
    for k in range(nv):
        ln = n >> k
        num, den = out[o:o + 2 * ln].reshape(-1, 2), out[o + 2 * ln:o + 4 * ln].reshape(-1, 2)
        layers.append((None if (mult is None and k == 0) else num, den))
        o += 4 * ln
    return layers


@pytest.mark.parametrize("name", ["lookup_nv2_1cols", "table_nv3_16cols", "lookup_nv3_ch_p_minus_1", "table_nv3_cols_alternating",
                                  "lookup_nv3_cols_zero_c_zero", "table_nv3_mult_p_minus_1", "lookup_nv3_ch_non_canonical"])
def test_reference_matches_the_oracle_circuit(name):
    case = LOGUP_BY_NAME[name]
    cols, mult, (c, g), _ = make_logup_inputs(case)
    exp, got = oracle_circuit(cols, mult, c, g), ref_circuit(cols, mult, c, g)
    assert len(exp) == len(got) == case.nv
    for k, ((en, ed), (gn, gd)) in enumerate(zip(exp, got)):
        assert (en is None) == (gn is None), k
        assert (ed == gd).all() and (en is None or (en == gn).all()), "layer %d" % k


# ---- device wrappers (C ABI, include/deepprove_b200.h) ---------------------------------------------------------------------
def _abi(gpu):
    L = gpu.lib()
    if not getattr(L, "_lookup_abi", False):
        L.dp_logup_build.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        L.dp_logup_num_vars.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]
        L.dp_logup_outputs.argtypes = [C.c_void_p, C.c_void_p]
        L.dp_logup_layer_mles.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
        L.dp_logup_free.argtypes = [C.c_void_p]
        L.dp_mle_linear_combination.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p)]
        L.dp_mle_evaluate_many.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
        L.dp_wit_matmul.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(C.c_void_p)]
        L._lookup_abi = True
    return L


def _handles(mles):
    return (C.c_void_p * max(1, len(mles)))(*[None if m is None else m.h for m in mles])


class Logup:
    def __init__(self, gpu, cols, mult, c, gamma, n_columns=None):
        self.gpu, self.L = gpu, _abi(gpu)
        self._c, self._g = O.u64(c), O.u64(gamma)
        self.h = C.c_void_p()
        gpu.check(self.L.dp_logup_build(_handles(cols), len(cols) if n_columns is None else n_columns,
                                        None if mult is None else mult.h, self._c.ctypes.data, self._g.ctypes.data, C.byref(self.h)))

    def num_vars(self):
        v = C.c_uint32()
        self.gpu.check(self.L.dp_logup_num_vars(self.h, C.byref(v)))
        return v.value

    def outputs(self):
        out = np.zeros(8, dtype=np.uint64)
        self.gpu.check(self.L.dp_logup_outputs(self.h, out.ctypes.data))
        return out.reshape(4, 2)

    def layer_views(self, layer_vars):
        views, n = (C.c_void_p * 4)(), C.c_uint32()
        self.gpu.check(self.L.dp_logup_layer_mles(self.h, layer_vars, views, C.byref(n)))
        return [self.gpu.Mle(views[i]).download() for i in range(n.value)]    # non-owning views: freeing one leaves the layer

    def free(self):
        if self.h:
            self.L.dp_logup_free(self.h)
            self.h = C.c_void_p()


def linear_combination(gpu, mles, coefs, n=None):
    cf = O.u64(coefs).reshape(-1)
    out = C.c_void_p()
    gpu.check(_abi(gpu).dp_mle_linear_combination(_handles(mles), cf.ctypes.data, len(mles) if n is None else n, C.byref(out)))
    return gpu.Mle(out.value)


def evaluate_many(gpu, mles, point, num_vars):
    pt = O.u64(point).reshape(-1)
    out = np.zeros(2 * len(mles), dtype=np.uint64)
    gpu.check(_abi(gpu).dp_mle_evaluate_many(_handles(mles), len(mles), pt.ctypes.data if pt.size else None, num_vars, out.ctypes.data))
    return out.reshape(-1, 2)


def matmul(gpu, left, right, bias, R, K, Cc, transposed):
    out = C.c_void_p()
    gpu.check(_abi(gpu).dp_wit_matmul(left.h, right.h, None if bias is None else bias.h, R, K, Cc, int(transposed), C.byref(out)))
    return gpu.Mle(out.value)


# ---- device runs: the LogUp circuit --------------------------------------------------------------------------------------
@pytest.fixture(scope="module", autouse=True)
def _module_leaves_spin_mode():
    yield
    import dpb200
    assert dpb200.lib().dp_get_wait_mode() == SPIN, "a test left the process in blocking wait mode"


@pytest.fixture(params=[SPIN, BLOCK], ids=["spin", "block"])
def wait_mode(gpu, request):
    """runs the test in spin and in blocking wait mode, then back to spin"""
    gpu.set_wait_mode(request.param)
    try:
        yield request.param
    finally:
        gpu.set_wait_mode(SPIN)


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


def check_circuit(gpu, case, cols, mult, ref_ch, sent_ch):
    exp = ref_circuit(cols, mult, *ref_ch)
    dcols = [gpu.Mle.upload(a, False) for a in cols]
    dm = None if mult is None else gpu.Mle.upload(mult, False)
    lg = Logup(gpu, dcols, dm, *sent_ch)
    try:
        assert lg.num_vars() == case.nv - 1
        for layer_vars in range(case.nv):
            num, den = exp[case.nv - 1 - layer_vars]
            h = 1 << layer_vars
            want = ([] if num is None else [num[:h], num[h:]]) + [den[:h], den[h:]]
            got = lg.layer_views(layer_vars)
            assert len(got) == len(want) == (2 if (layer_vars == case.nv - 1 and not case.table) else 4), (case.name, layer_vars)
            for j, (g, w) in enumerate(zip(got, want)):
                assert g.shape == w.shape and (g == w).all(), "%s: layer_vars %d view %d" % (case.name, layer_vars, j)
        assert (lg.outputs() == ref_outputs(exp)).all(), "%s: outputs" % case.name
    finally:
        lg.free()
    for d, a in zip(dcols, cols):
        assert (d.download() == a).all(), "%s: a column was modified" % case.name
    if dm is not None:
        assert (dm.download() == mult).all(), "%s: the multiplicities were modified" % case.name


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in LOGUP_CASES])
def test_logup_case(gpu, kernel_profile, name):
    """every layer's views, the outputs and the untouched inputs against the reference; launches per kernel against the plan"""
    case = LOGUP_BY_NAME[name]
    cols, mult, ref_ch, sent_ch = make_logup_inputs(case)
    check_circuit(gpu, case, cols, mult, ref_ch, sent_ch)
    got = {k: v[0] for k, v in gpu.profile_read().items() if k.startswith("k_logup")}
    assert got == expected_profile(case.nv, case.table), "%s: launches per kernel differ from logup_plan" % name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lookup_nv3_2cols", "lookup_nv12_16cols", "table_nv13_3cols"])
def test_logup_outputs_read_twice(gpu, wait_mode, name):
    """the outputs wait on the word the tail kernel publishes (dp_wait_flag, the poller in blocking mode); a second read is the same"""
    case = LOGUP_BY_NAME[name]
    cols, mult, ref_ch, sent_ch = make_logup_inputs(case)
    exp = ref_outputs(ref_circuit(cols, mult, *ref_ch))
    lg = Logup(gpu, [gpu.Mle.upload(a, False) for a in cols], None if mult is None else gpu.Mle.upload(mult, False), *sent_ch)
    try:
        first = lg.outputs()
        assert (first == exp).all() and (lg.outputs() == first).all()
    finally:
        lg.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lookup_nv14_3cols", "table_nv12_16cols"])
def test_logup_freed_while_tail_may_run(gpu, wait_mode, name):
    """dp_logup_free right after dp_logup_build waits for the tail kernel that still owns the pinned output block; the device and
    the allocator are fine afterwards"""
    case = LOGUP_BY_NAME[name]
    cols, mult, _, sent_ch = make_logup_inputs(case)
    lg = Logup(gpu, [gpu.Mle.upload(a, False) for a in cols], None if mult is None else gpu.Mle.upload(mult, False), *sent_ch)
    lg.free()
    ev, pt = O.splitmix_e(_seed(name) + 3, 1 << 12), O.splitmix_e(_seed(name) + 4, 12)
    assert (gpu.Mle.upload(ev, True).evaluate(pt) == O.evaluate(ev, True, pt)).all()


def _refused(gpu, fn, message):
    with pytest.raises(gpu.DpError) as e:
        fn()
    assert e.value.code == gpu.DP_ERR_INVALID and message in str(e.value), str(e.value)


@pytest.mark.gpu
def test_logup_refusals(gpu):
    f = lambda n, s=0: gpu.Mle.upload(O.splitmix_f(s, n), False)
    ch = ((1, 2), (3, 4))
    cols = [f(16, k) for k in range(17)]
    _refused(gpu, lambda: Logup(gpu, cols[:1], None, *ch, n_columns=0), "dp_logup_build: bad argument")
    _refused(gpu, lambda: Logup(gpu, cols, None, *ch), "dp_logup_build: bad argument")
    _refused(gpu, lambda: Logup(gpu, [cols[0], f(8)], None, *ch), "All sets of evaluations should be the same length")
    _refused(gpu, lambda: Logup(gpu, [cols[0], gpu.Mle.upload(O.splitmix_e(1, 16), True)], None, *ch),
             "All sets of evaluations should be the same length")
    _refused(gpu, lambda: Logup(gpu, [f(2), f(2, 1)], None, *ch), "need at least 4 evaluations")
    _refused(gpu, lambda: Logup(gpu, cols[:2], gpu.Mle.upload(O.splitmix_e(1, 16), True), *ch),
             "Multiplicities length was not equal to column evaluations length")
    _refused(gpu, lambda: Logup(gpu, cols[:2], f(8), *ch), "Multiplicities length was not equal to column evaluations length")
    _refused(gpu, lambda: Logup(gpu, [None, cols[1]], None, *ch), "dp_logup_build: null column")
    _refused(gpu, lambda: Logup(gpu, [cols[0], None], None, *ch), "dp_logup_build: null column")
    lg = Logup(gpu, cols[:2], None, *ch)
    try:
        assert lg.num_vars() == 3
        lg.layer_views(3)
        _refused(gpu, lambda: lg.layer_views(4), "One of the circuits was not the same size as the others")
    finally:
        lg.free()


# ---- device runs: the helpers the LogUp prover calls ----------------------------------------------------------------------
def _coef_set(n, seed):
    """the value-edge coefficients first, then random ones, one non-canonical (limb + p)"""
    r = [tuple(int(v) for v in x) for x in O.splitmix_e(seed, n)]
    cf = (EDGE_CHALLENGES + r)[:n]
    sent = list(cf)
    if n > 5:
        small = (int(r[5][0]) & 0x7FFFFFFF, int(r[5][1]) & 0x7FFFFFFF)
        cf[5], sent[5] = small, (small[0] + P, small[1] + P)
    return cf, sent


def _ext_table(pattern, n, seed):
    if pattern == "random":
        return O.splitmix_e(seed, n)
    v = np.full((n, 2), P - 1, dtype=np.uint64)
    if pattern == "alternating":
        v[0::2] = 0
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 16])
@pytest.mark.parametrize("nv", [0, 10, 13])
def test_linear_combination(gpu, n, nv):
    """out = sum_k coef_k m_k (same_poly.rs:91-110) against Python integers"""
    s = _seed("lincomb%d_%d" % (n, nv))
    tabs = [_ext_table(("random", "p_minus_1", "alternating")[k % 3], 1 << nv, s + k) for k in range(n)]
    cf, sent = _coef_set(n, s + 100)
    acc = (np.zeros(1 << nv, dtype=object), np.zeros(1 << nv, dtype=object))
    for t, c in zip(tabs, cf):
        t0, t1 = _ext_obj(t)
        acc = _vadd(acc, _vmul((np.full(1 << nv, c[0] % P, dtype=object), np.full(1 << nv, c[1] % P, dtype=object)), (t0, t1)))
    got = linear_combination(gpu, [gpu.Mle.upload(t, True) for t in tabs], sent).download()
    assert got.shape == (1 << nv, 2) and (got == _ext_u64(acc)).all()


@pytest.mark.gpu
def test_linear_combination_refusals(gpu):
    e = [gpu.Mle.upload(O.splitmix_e(k, 16), True) for k in range(17)]
    cf = [(1, 0)] * 17
    msg = "dp_mle_linear_combination: bad argument"
    _refused(gpu, lambda: linear_combination(gpu, e[:1], cf[:1], n=0), msg)
    _refused(gpu, lambda: linear_combination(gpu, e, cf), msg)
    msg = "operands must be Ext MLEs of equal length"
    _refused(gpu, lambda: linear_combination(gpu, [e[0], gpu.Mle.upload(O.splitmix_f(1, 16), False)], cf[:2]), msg)
    _refused(gpu, lambda: linear_combination(gpu, [e[0], gpu.Mle.upload(O.splitmix_e(1, 8), True)], cf[:2]), msg)
    _refused(gpu, lambda: linear_combination(gpu, [None, e[1]], cf[:2]), "dp_mle_linear_combination: null operand")
    _refused(gpu, lambda: linear_combination(gpu, [e[0], None], cf[:2]), "dp_mle_linear_combination: null operand")


@pytest.mark.gpu
@pytest.mark.parametrize("values", ["random", "edges"])
@pytest.mark.parametrize("nv", [0, 1, 10, 16, 17])
@pytest.mark.parametrize("n", [1, 16, 17, 33])
def test_evaluate_many(gpu, n, nv, values):
    """n MLEs at one point: batches of 16 per launch (mle.cu:380-385), one by one for num_vars 0 and > 16 (:369-371); Base and
    Ext mixed; value-edge tables and points"""
    s = _seed("evalmany%d_%d_%s" % (n, nv, values))
    mles = []
    for k in range(n):
        ext = k % 2 == 1
        pat = "random" if values == "random" else ("p_minus_1", "alternating", "random")[k % 3]
        t = _ext_table(pat, 1 << nv, s + k)
        mles.append((t if ext else np.ascontiguousarray(t[:, 0]), ext))
    if values == "random":
        pt = O.splitmix_e(s + 999, nv)
    else:
        pt = np.array([EDGE_CHALLENGES[(k * 3 + 1) % len(EDGE_CHALLENGES)] for k in range(nv)], dtype=np.uint64).reshape(-1, 2)
    got = evaluate_many(gpu, [gpu.Mle.upload(a, e) for a, e in mles], pt, nv)
    for k, (a, e) in enumerate(mles):
        assert (got[k] == O.evaluate(a, e, pt)).all(), "MLE %d of %d" % (k, n)


@pytest.mark.gpu
def test_evaluate_many_refusals(gpu):
    a, b = gpu.Mle.upload(O.splitmix_f(1, 16), False), gpu.Mle.upload(O.splitmix_f(2, 8), False)
    _refused(gpu, lambda: evaluate_many(gpu, [a, b], O.splitmix_e(3, 4), 4), "MLE size does not match the point")
    with pytest.raises(gpu.DpError) as e:
        gpu.check(_abi(gpu).dp_mle_evaluate_many(_handles([a]), 0, O.splitmix_e(3, 4).ctypes.data, 4, np.zeros(2, np.uint64).ctypes.data))
    assert e.value.code == gpu.DP_ERR_INVALID


# ---- device runs: the lookup-witness kernels (csrc/witness.cu) ------------------------------------------------------------
QMIN, QMAX = -127, 127                      # quantization/mod.rs:28-29
RANGE, RELU, CLAMP = 2, 0, 3                # TableType (lookup/context.rs:53-63)


def from_field(a):
    a = np.asarray(a, dtype=np.uint64)
    return [int(v) - P if int(v) > P // 2 else int(v) for v in a]


@pytest.mark.gpu
@pytest.mark.parametrize("ncols", [1, 2, 4, 64, 128])
@pytest.mark.parametrize("nrows", [1, 2, 8, 2048])
def test_dense(gpu, nrows, ncols):
    """Dense::op: bias + W x in signed integers; one column is k_wit_dense_small, 2 and 4 columns leave 1 and 2 lanes of a warp row
    busy; rows of +127 and -127 against inputs at +-127"""
    rng = np.random.default_rng(nrows * 1000 + ncols)
    w = rng.integers(-127, 128, size=(nrows, ncols)); b = rng.integers(-127, 128, size=nrows); x = rng.integers(-127, 128, size=ncols)
    x[0::2], x[1::2] = 127, -127
    w[0] = 127
    if nrows > 1:
        w[1] = -127
        w[-1, 0::2], w[-1, 1::2] = 127, -127      # every product +127 * 127 or -127 * -127: the largest sum
    b[0] = 127
    out = gpu.Witness.dense(gpu.Mle.upload(to_field(w.reshape(-1)), False), gpu.Mle.upload(to_field(b), False),
                            gpu.Mle.upload(to_field(x), False), nrows, ncols)
    assert (out.download() == to_field(w @ x + b)).all()


MATMUL_SHAPES = [(2, 2, 4), (2, 1, 4), (1, 1, 1), (4, 1, 2), (256, 4, 256), (64, 64, 1024)]   # power-of-two tensors


@pytest.mark.gpu
@pytest.mark.parametrize("values", ["int8", "wide"])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "no_bias"])
@pytest.mark.parametrize("transposed", [0, 1], ids=["B", "B_transposed"])
@pytest.mark.parametrize("shape", MATMUL_SHAPES, ids=["%dx%dx%d" % s for s in MATMUL_SHAPES])
def test_matmul(gpu, shape, transposed, bias, values):
    """MatMul::op (matrix_mul.rs:230-311): left [R][K] x right ([K][C], or [C][K] with TransposeB) + bias[C] on every row.
    "wide" operands reach |sum| > 2^32; the int8 ones include +-127 everywhere in one row and column"""
    R, K, Cc = shape
    rng = np.random.default_rng(R * 7 + K * 13 + Cc + 100 * transposed)
    lim = 127 if values == "int8" else 1 << 24
    left = rng.integers(-lim, lim + 1, size=(R, K)); mat = rng.integers(-lim, lim + 1, size=(K, Cc)); bv = rng.integers(-lim, lim + 1, size=Cc)
    left[0] = lim; mat[:, 0] = lim if values == "int8" else -lim
    exp = left @ mat + (bv if bias else 0)           # |sum| < 2^55: exact in int64
    if values == "wide":
        assert np.abs(exp).max() > 1 << 32
    right = mat.T if transposed else mat
    out = matmul(gpu, gpu.Mle.upload(to_field(left.reshape(-1)), False), gpu.Mle.upload(to_field(np.ascontiguousarray(right).reshape(-1)), False),
                 gpu.Mle.upload(to_field(bv), False) if bias else None, R, K, Cc, transposed)
    assert (out.download() == to_field(exp.reshape(-1))).all()


@pytest.mark.gpu
def test_matmul_refuses_bad_shapes(gpu):
    a = gpu.Mle.upload(to_field(np.ones(8, dtype=np.int64)), False)
    _refused(gpu, lambda: matmul(gpu, a, a, None, 2, 4, 4, 0), "Incompatible shape found for input matrix")
    _refused(gpu, lambda: matmul(gpu, a, a, a, 2, 4, 2, 0), "Incompatible shape found for input matrix")


def ref_requant(x, shift, fpm, ibits, csize):
    """Requant::op (requant.rs:472-482: |x| <= 2^intermediate_bit_size else error bit 1) and gen_lookup_witness (:225-284):
    tmp = x * fpm + 2^(shift-1), clamping input tmp >> shift, output clamped to [MIN, MAX], chunk j = (tmp & (2^shift - 1)) >> 8j
    & 255; the clamping table has rows -2^(csize-1) .. 2^(csize-1) - 1 (lookup/context.rs:210-222), else error bit 2"""
    cin, cout, chunks, err, clamp_idx = [], [], [[] for _ in range(shift // 8)], 0, []
    for v in x:
        if abs(v) > 1 << ibits:
            err |= 1
        tmp = v * fpm + (1 << (shift - 1))
        cl, masked = tmp >> shift, tmp & ((1 << shift) - 1)
        cin.append(cl); cout.append(min(max(cl, QMIN), QMAX))
        for j in range(shift // 8):
            chunks[j].append((masked >> (8 * j)) & 255)
        idx = cl + (1 << (csize - 1))
        if 0 <= idx < 1 << csize:
            clamp_idx.append(idx)
        else:
            err |= 2
    return cin, cout, chunks, err, clamp_idx


def _requant_params(shift, family):
    """fpm / 2^shift is 3/4 ("exact": tmp is a multiple of 2^shift for x = 2 mod 4) or a little above, with low bits set
    ("dense"); inputs up to 2^ibits keep tmp inside 63 bits and reach both clamps below shift 56"""
    fpm = 3 << (shift - 2)
    if family == "dense":
        fpm += int(O.splitmix_f(shift, 1)[0]) % (1 << (shift - 3)) | 1
    ibits = 10 if shift <= 48 else 6
    return fpm, ibits, ibits + 1


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["exact", "dense"])
@pytest.mark.parametrize("shift", [8, 16, 24, 32, 40, 48, 56])
def test_requant(gpu, shift, family):
    """every input from -2^ibits to 2^ibits (the bound itself is no error), 1 to 7 chunks; both clamps; exact multiples of 2^shift"""
    fpm, ibits, csize = _requant_params(shift, family)
    x = list(range(-(1 << ibits), (1 << ibits) + 1))
    x += [0] * ((1 << (len(x) - 1).bit_length()) - len(x))
    cin, cout, chunks, err, clamp_idx = ref_requant(x, shift, fpm, ibits, csize)
    assert err == 0
    if shift <= 48:
        assert min(cin) < QMIN and max(cin) > QMAX
    if family == "exact":
        zero = [v for v, *c in zip(x, *chunks) if not any(c)]
        assert min(zero) < 0 < max(zero)
    wit = gpu.Witness([(RANGE, 0), (CLAMP, csize)])
    cols = wit.requant(gpu.Mle.upload(to_field(x), False), shift, fpm, ibits, 1, 0)
    assert len(cols) == 2 + shift // 8
    assert from_field(cols[0].download()) == cin and from_field(cols[1].download()) == cout
    for j, c in enumerate(chunks):
        assert [int(v) for v in cols[2 + j].download()] == c, "chunk %d" % j
    mults, bits = wit.finish()
    assert bits == 0
    assert (mults[0].download() == np.bincount(np.concatenate(chunks).astype(np.int64), minlength=256)).all()
    assert (mults[1].download() == np.bincount(clamp_idx, minlength=1 << csize)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("v,bits", [(1 << 12, 0), (-(1 << 12), 0), ((1 << 12) + 1, 1), (-(1 << 12) - 1, 1)])
def test_requant_input_bound(gpu, v, bits):
    """error bit 1 exactly above |x| = 2^intermediate_bit_size (requant.rs:474-478); fpm = 1 keeps the clamping index in its table"""
    wit = gpu.Witness([(RANGE, 0), (CLAMP, 8)])
    wit.requant(gpu.Mle.upload(to_field([v, 0, 1, -1]), False), 16, 1, 12, 1, 0)
    assert wit.finish()[1] == bits


@pytest.mark.gpu
@pytest.mark.parametrize("v,ok", [(-9, False), (-8, True), (7, True), (8, False)])
def test_requant_clamp_table_ends(gpu, v, ok):
    """clamping size 4: indices 0 and 15 are the table's first and last rows, -1 and 16 are outside (error bit 2, not counted)"""
    shift = 8
    wit = gpu.Witness([(RANGE, 0), (CLAMP, 4)])
    wit.requant(gpu.Mle.upload(to_field([v, 0, 0, 0]), False), shift, 1 << shift, 20, 1, 0)
    mults, bits = wit.finish()
    assert bits == (0 if ok else 2)
    exp = np.zeros(16, dtype=np.uint64); exp[8] = 3
    if ok:
        exp[v + 8] += 1
    assert (mults[1].download() == exp).all()


@pytest.mark.gpu
@pytest.mark.parametrize("ibits", [63, 64, 1000])
def test_requant_refuses_intermediate_bits_above_62(gpu, ibits):
    wit = gpu.Witness([(RANGE, 0), (CLAMP, 8)])
    x = gpu.Mle.upload(to_field([1, 2, 3, 4]), False)
    _refused(gpu, lambda: wit.requant(x, 16, 3 << 14, ibits, 1, 0), "intermediate_bit_size must be at most 62")
    wit.requant(x, 16, 3 << 14, 62, 1, 0)


@pytest.mark.gpu
def test_relu_every_table_row_and_the_ends(gpu):
    """the Relu table's rows are x = MIN - 1 .. MAX (lookup/context.rs:182-199); each counted once, out = max(x, 0)
    (activation.rs:265-279); then -129 and 128 fall outside it (error bit 4) and add nothing"""
    x = list(range(QMIN - 1, QMAX + 1))
    wit = gpu.Witness([(RELU, 0)])
    out = wit.relu(gpu.Mle.upload(to_field(x), False), 0)
    assert from_field(out.download()) == [max(v, 0) for v in x]
    mults, bits = wit.finish()
    assert bits == 0 and (mults[0].download() == 1).all()
    wit = gpu.Witness([(RELU, 0)])
    y = [QMIN - 2, QMAX + 1, QMAX, QMIN - 1] * 4
    out = wit.relu(gpu.Mle.upload(to_field(y), False), 0)
    assert from_field(out.download()) == [max(v, 0) for v in y]
    mults, bits = wit.finish()
    exp = np.zeros(256, dtype=np.uint64); exp[0] = exp[255] = 4
    assert bits == 4 and (mults[0].download() == exp).all()


def ref_pool(t):
    """Maxpool2D (kernel = stride = 2, pooling.rs:667-676) and its difference columns out - in(2r+dr, 2c+dc) for
    (dr, dc) = (0,0), (1,0), (0,1), (1,1) (compute_polys, :686-768); a difference above 255 is outside the range table"""
    Cn, H, W = t.shape
    win = t.reshape(Cn, H // 2, 2, W // 2, 2)
    mx = win.max(axis=(2, 4))
    diffs = [(mx - win[:, :, dr, :, dc]).reshape(-1) for dr, dc in ((0, 0), (1, 0), (0, 1), (1, 1))]
    return mx.reshape(-1), diffs


POOL_SHAPES = [(1, 2, 2), (2, 4, 8), (4, 8, 2), (8, 16, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("values", ["negative_ties", "diff_255"])
@pytest.mark.parametrize("shape", POOL_SHAPES, ids=["%dx%dx%d" % s for s in POOL_SHAPES])
def test_pool(gpu, shape, values):
    rng = np.random.default_rng(sum(shape))
    if values == "negative_ties":
        t = rng.integers(-128, 1, size=shape)
        t[..., 0::2, :] = t[..., 1::2, :]                # every window has a tie
    else:
        t = rng.integers(-128, 128, size=shape)
        t[0, 0, 0], t[0, 1, 1] = 127, -128              # one window spans exactly 255
    mx, diffs = ref_pool(t)
    wit = gpu.Witness([(RANGE, 0)])
    cols = wit.pool(gpu.Mle.upload(to_field(t.reshape(-1)), False), *shape, 0)
    assert from_field(cols[4].download()) == [int(v) for v in mx]
    for k in range(4):
        assert [int(v) for v in cols[k].download()] == [int(v) for v in diffs[k]], "column %d" % k
    mults, bits = wit.finish()
    all_d = np.concatenate(diffs)
    assert bits == 0 and (values != "diff_255" or all_d.max() == 255)
    assert (mults[0].download() == np.bincount(all_d, minlength=256)).all()


@pytest.mark.gpu
def test_pool_difference_256_is_an_error(gpu):
    """windows [100, -156; 100, 100] (a difference of 256: error bit 8, not counted) and [0, 0; 3, 100]"""
    t = np.array([100, -156, 0, 0, 100, 100, 3, 100], dtype=np.int64).reshape(1, 2, 4)
    mx, diffs = ref_pool(t)
    wit = gpu.Witness([(RANGE, 0)])
    cols = wit.pool(gpu.Mle.upload(to_field(t.reshape(-1)), False), 1, 2, 4, 0)
    assert from_field(cols[4].download()) == [int(v) for v in mx] == [100, 100]
    mults, bits = wit.finish()
    d = np.concatenate(diffs)
    assert sorted(d.tolist()) == [0, 0, 0, 0, 97, 100, 100, 256]
    assert bits == 8 and (mults[0].download() == np.bincount(d[d <= 255], minlength=256)).all()


def _requant_node(wit, gpu, x, shift, fpm, ibits, tables, clamp_table, range_table):
    wit.requant(gpu.Mle.upload(to_field(x), False), shift, fpm, ibits, clamp_table, range_table)
    return ref_requant(x, shift, fpm, ibits, tables[clamp_table][1])


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["one_table", "three_tables", "eight_tables"])
def test_finish_several_nodes_into_shared_tables(gpu, layout):
    """histograms that several node calls add into, tables of every kind in one witness (clamping sizes 1 and 24 included), error
    bits OR-ed across nodes"""
    tables = {"one_table": [(RANGE, 0)],
              "three_tables": [(CLAMP, 11), (RANGE, 0), (RELU, 0)],
              "eight_tables": [(RELU, 0), (CLAMP, 1), (RANGE, 0), (CLAMP, 24), (CLAMP, 11), (RANGE, 0), (RELU, 0), (CLAMP, 9)]}[layout]
    wit = gpu.Witness(tables)
    exp = [np.zeros(1 << (s if k == CLAMP else 8), dtype=np.int64) for k, s in tables]
    rng_t = [i for i, (k, _) in enumerate(tables) if k == RANGE]
    err = 0
    rng = np.random.default_rng(len(tables))
    if layout == "one_table":
        for shape in ((1, 4, 4), (2, 4, 8)):
            t = rng.integers(-128, 128, size=shape)
            wit.pool(gpu.Mle.upload(to_field(t.reshape(-1)), False), *shape, 0)
            exp[0] += np.bincount(np.concatenate(ref_pool(t)[1]), minlength=256)
    else:
        clamps = [i for i, t in enumerate(tables) if t in ((CLAMP, 24), (CLAMP, 11))]
        relus = [i for i, (k, _) in enumerate(tables) if k == RELU]
        nodes = [(list(range(-1024, 1024)), 16), (rng.integers(-1024, 1025, size=512).tolist(), 24)]
        for j, (x, shift) in enumerate(nodes):      # two requants into the same range table, clamping tables of 2^11 and 2^9 rows
            ct, rt = clamps[j % len(clamps)], rng_t[0]
            fpm = 3 << (shift - 2) if tables[ct][1] == 11 else 1 << (shift - 2)
            _, _, chunks, e, idx = _requant_node(wit, gpu, x, shift, fpm, 10, tables, ct, rt)
            err |= e
            exp[rt] += np.bincount(np.concatenate(chunks).astype(np.int64), minlength=256)
            exp[ct] += np.bincount(idx, minlength=len(exp[ct])).astype(np.int64)
        t = rng.integers(-128, 128, size=(2, 4, 4))      # a pool into the same range table
        wit.pool(gpu.Mle.upload(to_field(t.reshape(-1)), False), 2, 4, 4, rng_t[0])
        exp[rng_t[0]] += np.bincount(np.concatenate(ref_pool(t)[1]), minlength=256)
        for r in relus:                                  # relus, one with a value outside its table
            y = rng.integers(-128, 128, size=63).tolist() + [200]
            wit.relu(gpu.Mle.upload(to_field(y), False), r)
            exp[r] += np.bincount([v + 128 for v in y if -128 <= v <= 127], minlength=256)
            err |= 4
        if layout == "eight_tables":
            small = tables.index((CLAMP, 1))             # clamping size 1: rows -1 and 0
            _, _, chunks, e, idx = _requant_node(wit, gpu, [-1, 0, 0, -1], 8, 1 << 8, 4, tables, small, rng_t[1])
            exp[small] += np.bincount(idx, minlength=2); exp[rng_t[1]] += np.bincount(np.concatenate(chunks).astype(np.int64), minlength=256)
            big = tables.index((CLAMP, 24))              # clamping size 24: the first and last rows
            x = [-(1 << 23), (1 << 23) - 1, 0, 1 << 24]  # the last is too large for intermediate_bit_size 23: error bit 1 (and 2)
            _, _, chunks, e, idx = _requant_node(wit, gpu, x, 8, 1 << 8, 23, tables, big, rng_t[1])
            assert e == 3
            err |= e
            exp[big] += np.bincount(idx, minlength=1 << 24); exp[rng_t[1]] += np.bincount(np.concatenate(chunks).astype(np.int64), minlength=256)
    mults, bits = wit.finish()
    assert len(mults) == len(tables) and bits == err
    for i, (m, e) in enumerate(zip(mults, exp)):
        assert (m.download() == e.astype(np.uint64)).all(), "table %d %s" % (i, tables[i])


@pytest.mark.gpu
def test_witness_refusals(gpu):
    msg = "dp_wit_begin: 1..8 tables"
    _refused(gpu, lambda: gpu.Witness([]), msg)
    _refused(gpu, lambda: gpu.Witness([(RANGE, 0)] * 9), msg)
    for t in ((1, 0), (CLAMP, 0), (CLAMP, 25)):
        _refused(gpu, lambda: gpu.Witness([(RANGE, 0), t]), "dp_wit_begin: unknown table type")
    wit = gpu.Witness([(RANGE, 0), (CLAMP, 8), (RELU, 0)])
    x = gpu.Mle.upload(to_field([1, 2, 3, 4]), False)
    _refused(gpu, lambda: wit.requant(x, 8, 1, 10, 0, 0), "dp_wit_requant: wrong table index/type")
    _refused(gpu, lambda: wit.requant(x, 8, 1, 10, 1, 3), "dp_wit_requant: wrong table index/type")
    _refused(gpu, lambda: wit.relu(x, 1), "dp_wit_relu: wrong table index/type")
    _refused(gpu, lambda: wit.relu(x, 3), "dp_wit_relu: wrong table index/type")
    _refused(gpu, lambda: wit.pool(x, 1, 2, 2, 2), "dp_wit_pool: wrong table index/type")
    mults, bits = wit.finish()
    assert bits == 0 and all((m.download() == 0).all() for m in mults)
