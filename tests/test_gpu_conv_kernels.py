"""The FFT-convolution kernels (deep-prove_b200/csrc/conv.cu) against a big-integer reference, kernel by kernel, at every row
length and at value edges.

The reference restates each operation in Python integers mod p = 2^64 - 2^32 + 1, with E = F[X]/(X^2 - 7): fft (tensor.rs:261-323),
index_w / index_wf (dp_pad_rows), index_x's row reversal (dp_reverse_rows), fft_conv's accumulation (dp_conv_prod), index_u +
to_element + add_bias (dp_conv_output_elements / dp_conv_output), phi_pow_init / phi_g_init (iop/prover.rs:215-284, every `mid`
table), one delegate_matrix_evaluation phi level (dp_phi_level) and beta_acc's repeat (dp_mle_repeat).  CPU tests pin the
reference to the naive DFT, to the closed form of phi_g_init and to the CPU checker (oracle/); the GPU tests compare every output
word with it and read dp_kernel_launches to confirm the path each call takes.  Rows longer than 2^13 and phi tables above 2^15 are
too large for Python integers: there the closed-form patterns (constants, impulses), the checker's fft, and phi_g_init's same
steps on the checker's vectorised field operations, all pinned to the reference by the CPU tests, stand in.
"""
import ctypes as C
import functools
import glob
import os
import re
import zlib

import numpy as np
import pytest

import oracle_py as O
from test_launch_rule import strip_comments

P = O.P
HALF = P >> 1
ROOT_2_32 = 1753635133440165772   # Goldilocks two_adic_generator(32): get_root_of_unity(n) = ROOT_2_32^(2^(32 - n)) (tensor.rs:220-231)
ZERO, ONE = (0, 0), (1, 0)
EDGES = [(0, 0), (1, 0), (P - 1, 0), (P - 1, P - 1), (0, 1)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "deep-prove_b200", "csrc")


def _seed(*key):
    return zlib.crc32(repr(key).encode()) & 0xFFFFFF


# ---- Ext arithmetic: an Ext vector is a pair (c0, c1) of object arrays of Python ints; an Ext scalar a pair of ints ----------
def ext(a):
    a = np.asarray(a, dtype=np.uint64).reshape(-1, 2)
    return a[:, 0].astype(object), a[:, 1].astype(object)


def u64e(v):
    """an Ext vector (or a list of Ext scalars) as the [n, 2] words the device stores"""
    if isinstance(v, list):
        return np.array(v, dtype=np.uint64).reshape(-1, 2)
    return np.stack([np.asarray(v[0] % P, dtype=object).astype(np.uint64).reshape(-1),
                     np.asarray(v[1] % P, dtype=object).astype(np.uint64).reshape(-1)], axis=1)


def vmul(a, b):
    """(a0 + a1 X)(b0 + b1 X) with X^2 = 7"""
    return (a[0] * b[0] + 7 * a[1] * b[1]) % P, (a[0] * b[1] + a[1] * b[0]) % P


def vadd(a, b):
    return (a[0] + b[0]) % P, (a[1] + b[1]) % P


def vsub(a, b):
    return (a[0] - b[0]) % P, (a[1] - b[1]) % P


def vscale(a, s):
    """an Ext times a base-field value"""
    return a[0] * s % P, a[1] * s % P


def inv(x):
    return pow(x, P - 2, P)


def root(log_n):
    return pow(ROOT_2_32, 1 << (32 - log_n), P)


def rand_e(seed, n):
    return O.splitmix_e(seed, n)


# ---- fft (tensor.rs:261-323) -------------------------------------------------------------------------------------------------
def ref_fft(v, inverse=False):
    """natural order in and out; w = get_root_of_unity(log n), inverted for the iFFT, which also scales by 1/n"""
    c0, c1 = (np.array(x, dtype=object) for x in v)
    n = len(c0)
    logn = n.bit_length() - 1
    rev = [0] * n
    for i in range(1, n):
        rev[i] = rev[i >> 1] >> 1 | (i & 1) << (logn - 1)
    w1 = root(logn)
    if inverse:
        w1 = inv(w1)
    w = [1] * n
    for i in range(1, n):
        w[i] = w[i - 1] * w1 % P
    c0, c1 = c0[rev], c1[rev]                     # the swaps of i and rev[i] < i: rev is an involution
    i = 2
    while i <= n:
        h = i >> 1
        tw = np.array([w[n // i * k] for k in range(h)], dtype=object)
        a0, a1 = c0.reshape(-1, i), c1.reshape(-1, i)
        u0, u1 = a0[:, :h].copy(), a1[:, :h].copy()
        l0, l1 = a0[:, h:] * tw % P, a1[:, h:] * tw % P
        a0[:, :h], a0[:, h:] = (u0 + l0) % P, (u0 - l0) % P
        a1[:, :h], a1[:, h:] = (u1 + l1) % P, (u1 - l1) % P
        i <<= 1
    if inverse:
        return vscale((c0, c1), inv(n))
    return c0, c1


def naive_dft(v, inverse=False):
    c0, c1 = (list(map(int, x)) for x in v)
    n = len(c0)
    w = root(n.bit_length() - 1)
    if inverse:
        w = inv(w)
    out0, out1 = [], []
    for k in range(n):
        s0 = s1 = 0
        for j in range(n):
            t = pow(w, j * k, P)
            s0, s1 = s0 + c0[j] * t, s1 + c1[j] * t
        out0.append(s0 % P)
        out1.append(s1 % P)
    o = (np.array(out0, dtype=object), np.array(out1, dtype=object))
    return vscale(o, inv(n)) if inverse else o


@functools.lru_cache(maxsize=2)
def pow_table(log_n, inverse):
    """w^e for e < n as words, w = get_root_of_unity(log n); for the inverse, w^-e / n"""
    n = 1 << log_n
    w = inv(root(log_n)) if inverse else root(log_n)
    x = inv(n) if inverse else 1
    out = [0] * n
    for e in range(n):
        out[e] = x
        x = x * w % P
    return np.array(out, dtype=np.uint64)


def impulse_transform(log_n, j, inverse):
    """the transform of delta_j: X[k] = w^(jk) (forward), w^(-jk) / n (inverse) -- a geometric sequence"""
    n = 1 << log_n
    out = np.zeros((n, 2), dtype=np.uint64)
    out[:, 0] = pow_table(log_n, inverse)[(np.uint64(j) * np.arange(n, dtype=np.uint64)) % np.uint64(n)]
    return out


def impulse_points(log_n):
    """0, 1, n - 1 and both sides of the four-step splits N1 = 2^(log n / 2) and N2 = n / N1"""
    n, n1 = 1 << log_n, 1 << (log_n // 2)
    n2 = n // n1
    return sorted({j for j in (0, 1, n - 1, n2 - 1, n2, n1 - 1, n1) if 0 <= j < n})


def _constant(n, c, scale):
    out = np.zeros((n, 2), dtype=np.uint64)
    out[0] = (scale * c[0] % P, scale * c[1] % P)
    return out


def fft_patterns(log_n):
    """[(name, row(), transform(inverse))]: the transforms in closed form, the random row's from the checker's fft.  Built on
    demand: at 2^21 each row is 32 MB."""
    n = 1 << log_n
    pats = [("zeros", lambda: np.zeros((n, 2), dtype=np.uint64), lambda inverse: np.zeros((n, 2), dtype=np.uint64))]
    for name, c in (("p-1", (P - 1, 0)), ("(p-1,p-1)", (P - 1, P - 1)), ("ones", ONE)):
        # n equal values: n c at k = 0 (forward) or c there (inverse), 0 elsewhere
        pats.append((name, lambda c=c: np.tile(np.array(c, dtype=np.uint64), (n, 1)),
                     lambda inverse, c=c: _constant(n, c, 1 if inverse else n)))
    for j in impulse_points(log_n):
        def row(j=j):
            r = np.zeros((n, 2), dtype=np.uint64)
            r[j, 0] = 1
            return r
        pats.append(("delta_%d" % j, row, lambda inverse, j=j: impulse_transform(log_n, j, inverse)))
    rand = functools.lru_cache(maxsize=1)(lambda: rand_e(_seed("fft", log_n), n))
    pats.append(("random", rand, lambda inverse: O.fft_ext(rand()[None], inverse=inverse)[0]))
    return pats


def random_pattern(log_n, i):
    row = rand_e(_seed("fft extra", log_n, i), 1 << log_n)
    return ("random %d" % i, lambda: row, lambda inverse: O.fft_ext(row[None], inverse=inverse)[0])


# ---- phi_pow_init / phi_g_init (iop/prover.rs:215-284) -------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def ref_phi_pow_init(n, is_fft):
    """phi_mul[i] = phi^i, phi = get_root_of_unity(n), inverted when is_fft"""
    phi = root(n)
    if is_fft:
        phi = inv(phi)
    out = [1] * (1 << n)
    for i in range(1, 1 << n):
        out[i] = out[i - 1] * phi % P
    return np.array(out, dtype=object)


def ref_phi_g_init(rx, scale, n, is_fft):
    """prover.rs:231-284 literally, one level at a time: returns phi_g and mid[0 .. n - 2] as Ext vectors"""
    phi_mul = ref_phi_pow_init(n, bool(is_fft))
    g = [np.zeros(1 << n, dtype=object), np.zeros(1 << n, dtype=object)]
    g[0][0], g[1][0] = scale
    if is_fft:
        g[0][1], g[1][1] = scale
    mid = []
    for i in range(1, (n + 1) if is_fft else n):
        cnt, m = 1 << (i - 1), n - i
        tmp1 = vsub(ONE, rx[m])
        tmp2 = vscale(rx[m], phi_mul[::1 << m][:cnt])          # rx[m] * phi_mul[b << m]
        left = (g[0][:cnt].copy(), g[1][:cnt].copy())
        g[0][cnt:2 * cnt], g[1][cnt:2 * cnt] = vmul(left, vsub(tmp1, tmp2))
        g[0][:cnt], g[1][:cnt] = vmul(left, vadd(tmp1, tmp2))
        if i < n:
            mid.append((g[0][:2 * cnt].copy(), g[1][:2 * cnt].copy()))
    if not is_fft:
        h = 1 << (n - 1)
        g[0][:h], g[1][:h] = vmul((g[0][:h], g[1][:h]), vadd(vsub(ONE, rx[0]), vscale(rx[0], phi_mul[:h])))
    return (g[0], g[1]), mid


def closed_phi_g(rx, scale, n, is_fft, levels):
    """scale * prod_{m in [n - levels, n)} (1 - rx[m] + rx[m] phi^(j 2^m)) for j < 2^levels (j < 2^(n - 1) when the iFFT's table
    is complete, its top half 0); phi = w^-1 for the FFT and w for the iFFT"""
    phi = inv(root(n)) if is_fft else root(n)
    size = 1 << levels
    top = size if (is_fft or levels < n) else size >> 1
    out = []
    for j in range(size):
        v = scale if j < top else ZERO
        if j < top:
            for m in range(n - levels, n):
                v = vmul(v, vadd(vsub(ONE, rx[m]), vscale(rx[m], pow(phi, j << m, P))))
        out.append(v)
    return out


def _fill(e, n):
    return np.tile(np.array(e, dtype=np.uint64), (n, 1))


def _lift(base):
    return np.stack([base, np.zeros_like(base)], axis=1)


def fast_phi_pow_init(n, is_fft):
    """ref_phi_pow_init as words, by doubling: phi^(i + 2^k) = phi^i * phi^(2^k)"""
    phi = inv(root(n)) if is_fft else root(n)
    out = np.ones(1, dtype=np.uint64)
    while out.size < (1 << n):
        out = np.concatenate([out, O.f_binop(2, out, np.full(out.size, phi, dtype=np.uint64))])
        phi = phi * phi % P
    return out


def fast_phi_g_init(rx, scale, n, is_fft):
    """ref_phi_g_init step for step on [len, 2] words, with the checker's vectorised field operations (oracle_py.e_binop: 0 add,
    1 sub, 2 mul) in place of Python integers, which take seconds per table above 2^15"""
    phi_mul = fast_phi_pow_init(n, bool(is_fft))
    g = np.zeros((1 << n, 2), dtype=np.uint64)
    g[0] = scale
    if is_fft:
        g[1] = scale
    mid = []
    for i in range(1, (n + 1) if is_fft else n):
        cnt, m = 1 << (i - 1), n - i
        tmp1 = _fill(vsub(ONE, rx[m]), cnt)
        tmp2 = O.e_binop(2, _fill(rx[m], cnt), _lift(phi_mul[::1 << m][:cnt]))
        left = g[:cnt].copy()
        g[cnt:2 * cnt] = O.e_binop(2, left, O.e_binop(1, tmp1, tmp2))
        g[:cnt] = O.e_binop(2, left, O.e_binop(0, tmp1, tmp2))
        if i < n:
            mid.append(g[:2 * cnt].copy())
    if not is_fft:
        h = 1 << (n - 1)
        g[:h] = O.e_binop(2, g[:h], O.e_binop(0, _fill(vsub(ONE, rx[0]), h), O.e_binop(2, _fill(rx[0], h), _lift(phi_mul[:h]))))
    return g, mid


def phi_inputs(case, n):
    """(rx, scale) for a named case: random, or edge values 0, 1, p - 1, (p - 1, p - 1), (0, 1) in rx and scale"""
    r = [tuple(map(int, e)) for e in rand_e(_seed("rx", case, n), n + 1)]
    rx, scale = r[:n], r[n]
    if case == "rx edges":
        rx = [EDGES[m % len(EDGES)] for m in range(n)]
    elif case == "rx edges mixed, scale p-1":
        rx = [EDGES[m % len(EDGES)] if m % 2 else rx[m] for m in range(n)]
        scale = (P - 1, P - 1)
    elif case == "scale 0":
        scale = ZERO
    elif case == "rx (0,1), scale 1":
        rx, scale = [(0, 1)] * n, ONE
    return rx, scale


PHI_CASES = ["random", "rx edges", "rx edges mixed, scale p-1", "scale 0", "rx (0,1), scale 1"]


# ---- one delegate_matrix_evaluation level (prover.rs:182-195) ------------------------------------------------------------------
def ref_phi_level(len_log, n_total, shift, A, B, inverse):
    """phi[i] = A + B * omegas[i << shift], omegas = phi_pow_init(n_total, inverse)"""
    w = inv(root(n_total)) if inverse else root(n_total)
    return [vadd(A, vscale(B, pow(w, (i << shift) % (1 << n_total), P))) for i in range(1 << len_log)]


# ---- the layer's tensors ----------------------------------------------------------------------------------------------------
def ref_pad_rows(src, rows, n_real, n, out_len):
    """index_w / index_wf: each n_real x n_real block top-left in an n x n grid, the row zero-padded to out_len (Base lifted)"""
    src = np.asarray(src, dtype=np.uint64)
    src = src.reshape(rows, n_real * n_real, -1)
    out = np.zeros((rows, out_len, 2), dtype=np.uint64)
    for idx in range(min(out_len, n * n_real)):
        i, j = divmod(idx, n)
        if i < n_real and j < n_real:
            out[:, idx, :src.shape[2]] = src[:, i * n_real + j]
    return out.reshape(-1, 2)


def ref_reverse_rows(src, row_len):
    """index_x's reversal of every row (tensor.rs:343-361)"""
    return np.asarray(src).reshape(-1, row_len)[:, ::-1].reshape(-1)


def ref_conv_prod(x, w, kw, kx, n):
    """fft_conv's accumulation (tensor.rs:489-509): out[i][k] = sum_j x[j][k] * w[i][j][k]"""
    xv, wv = ext(x), ext(w)
    out0, out1 = [], []
    for i in range(kw):
        acc = (np.zeros(n, dtype=object), np.zeros(n, dtype=object))
        for j in range(kx):
            xj = (xv[0][j * n:(j + 1) * n], xv[1][j * n:(j + 1) * n])
            wij = (wv[0][(i * kx + j) * n:(i * kx + j + 1) * n], wv[1][(i * kx + j) * n:(i * kx + j + 1) * n])
            acc = vadd(acc, vmul(xj, wij))
        out0.append(acc[0])
        out1.append(acc[1])
    return u64e((np.concatenate(out0), np.concatenate(out1)))


def to_element(c0, c1):
    """quantization/mod.rs:225-242"""
    if c0 == 0 and c1 == 0:
        return 0
    return c0 if c0 <= HALF else -(P - c0)


def ref_conv_output_elements(rows, kw, n_x, bias):
    """index_u + to_element + add_bias: out[i][t] = to_element(rows[i][n_x^2 - 1 - t]) + bias[i]"""
    nx2 = n_x * n_x
    r = np.asarray(rows, dtype=np.uint64).reshape(kw, 2 * nx2, 2)
    return np.array([[to_element(int(r[i, nx2 - 1 - t, 0]), int(r[i, nx2 - 1 - t, 1])) + int(bias[i]) for t in range(nx2)]
                     for i in range(kw)], dtype=np.int64).reshape(-1)


def ref_conv_output(rows, kw, n_x, bias_f, mask):
    """the same tensor as field elements, after = c0 + bias, and cleared = after * mask"""
    nx2 = n_x * n_x
    r = np.asarray(rows, dtype=np.uint64).reshape(kw, 2 * nx2, 2)
    c0 = r[:, nx2 - 1::-1, 0].astype(object)                                    # rows[i][n_x^2 - 1 - t].c0
    after = (c0 + np.asarray(bias_f, dtype=np.uint64).astype(object)[:, None]) % P
    cleared = after * np.asarray(mask, dtype=np.uint64).reshape(kw, nx2).astype(object) % P
    return after.reshape(-1).astype(np.uint64), cleared.reshape(-1).astype(np.uint64)


def field(v):
    """an int64 vector as canonical field words"""
    return np.array([int(x) % P for x in v], dtype=np.uint64)


# ================================================ CPU: the reference pinned ===================================================
def test_root_has_order_2_32():
    assert pow(ROOT_2_32, 1 << 32, P) == 1 and pow(ROOT_2_32, 1 << 31, P) == P - 1


@pytest.mark.parametrize("log_n", range(1, 7))
def test_fft_equals_naive_dft(log_n):
    n = 1 << log_n
    v = ext(rand_e(_seed("dft", log_n), n))
    for inverse in (False, True):
        got, exp = ref_fft(v, inverse), naive_dft(v, inverse)
        assert all((got[c] == exp[c]).all() for c in (0, 1))
    back = ref_fft(ref_fft(v), inverse=True)
    assert all((back[c] == v[c]).all() for c in (0, 1))


@pytest.mark.parametrize("log_n", range(1, 14))
def test_fft_equals_the_checker(log_n):
    """the restated fft equals oracle_py.fft_ext, which the GPU tests use for rows too long for Python integers"""
    v = rand_e(_seed("fft oracle", log_n), 1 << log_n)
    for inverse in (False, True):
        assert (u64e(ref_fft(ext(v), inverse)) == O.fft_ext(v[None], inverse=inverse)[0]).all()


@pytest.mark.parametrize("log_n", range(1, 9))
def test_fft_closed_forms(log_n):
    """every closed-form pattern the long-row GPU tests use equals the restated fft of its row"""
    for name, row, transform in fft_patterns(log_n):
        for inverse in (False, True):
            assert (u64e(ref_fft(ext(row()), inverse)) == transform(inverse)).all(), (name, inverse)


@pytest.mark.parametrize("n", range(2, 9))
@pytest.mark.parametrize("is_fft", [1, 0])
@pytest.mark.parametrize("case", PHI_CASES)
def test_phi_g_init_closed_form(n, is_fft, case):
    """phi_g[j] = scale * prod_{m<n} (1 - rx[m] + rx[m] phi^(j 2^m)), the iFFT's top half 0, and mid[i - 1] the same product over
    m in [n - i, n)"""
    rx, scale = phi_inputs(case, n)
    phi_g, mid = ref_phi_g_init(rx, scale, n, is_fft)
    assert (u64e(phi_g) == u64e(closed_phi_g(rx, scale, n, is_fft, n))).all()
    assert len(mid) == n - 1
    for i in range(1, n):
        assert (u64e(mid[i - 1]) == u64e(closed_phi_g(rx, scale, n, is_fft, i))).all(), i


@pytest.mark.parametrize("n", range(2, 17))
@pytest.mark.parametrize("is_fft", [1, 0])
def test_fast_phi_g_init_equals_the_restatement(n, is_fft):
    """the same steps on the checker's field operations, which the GPU tests use for tables above 2^15, give the Python-integer
    restatement's phi_g and mid tables"""
    for case in PHI_CASES:
        rx, scale = phi_inputs(case, n)
        phi_g, mid = ref_phi_g_init(rx, scale, n, is_fft)
        f_phi, f_mid = fast_phi_g_init(rx, scale, n, is_fft)
        assert (u64e(phi_g) == f_phi).all(), case
        assert len(f_mid) == n - 1 and all((u64e(a) == b).all() for a, b in zip(mid, f_mid)), case


@pytest.mark.parametrize("n_total", [1, 2, 5, 10])
def test_phi_level_is_a_slice_of_phi_pow_init(n_total):
    A, B = tuple(map(int, rand_e(3, 1)[0])), tuple(map(int, rand_e(4, 1)[0]))
    for inverse in (0, 1):
        omegas = ref_phi_pow_init(n_total, bool(inverse))
        for len_log in range(n_total + 1):
            for shift in range(n_total - len_log + 1):
                exp = [vadd(A, vscale(B, omegas[i << shift])) for i in range(1 << len_log)]
                assert ref_phi_level(len_log, n_total, shift, A, B, inverse) == exp


def test_to_element_sign_boundary():
    assert [to_element(c, 0) for c in (0, 1, HALF, HALF + 1, P - 1)] == [0, 1, HALF, -HALF, -1]
    assert to_element(0, 5) == 0


@pytest.mark.parametrize("values", ["random", "extreme", "alternating"])
def test_reference_layer_equals_the_checker(values):
    """index_x, pad, fft, the accumulation, the iFFT, index_u, to_element and the bias, composed, give the checker's conv_op"""
    kw, kx, n_x, rn = 2, 2, 8, 4
    filt, bias, x, uo = extreme_conv(values)
    nx2 = n_x * n_x
    xr = ref_reverse_rows(field(x.reshape(-1)), nx2)
    x_fft = np.concatenate([u64e(ref_fft(ext(ref_pad_rows(xr[c * nx2:(c + 1) * nx2], 1, n_x, n_x, 2 * nx2)))) for c in range(kx)])
    wp = ref_pad_rows(field(filt.reshape(-1)), kw * kx, rn, n_x, 2 * nx2)
    w_fft = np.concatenate([u64e(ref_fft(ext(wp[r * 2 * nx2:(r + 1) * 2 * nx2]))) for r in range(kw * kx)])
    prod = ref_conv_prod(x_fft, w_fft, kw, kx, 2 * nx2)
    rows = np.concatenate([u64e(ref_fft(ext(prod[i * 2 * nx2:(i + 1) * 2 * nx2]), inverse=True)) for i in range(kw)])
    after, _ = O.conv_op(filt, bias, uo, x)
    assert (ref_conv_output_elements(rows, kw, n_x, bias) == after.reshape(-1)).all()


def extreme_conv(values):
    """a 2 x 2 x 8 x 8 layer with 3 x 3 filters on 7 x 7 images: every weight -128 and every input 127, or random extremes so
    outputs take both signs; biases at the ends of a 32-bit accumulator"""
    filt, bias, x, uo = O.synthetic_conv(2, 2, 8, 4, 2, 3, 2, 7, 61, 62)
    rng = np.random.default_rng(_seed("extreme", values))
    if values == "extreme":
        filt[:, :, :3, :3] = -128
        x[:, :7, :7] = 127
        bias[:] = (1 << 31) - 1, -(1 << 31)
    elif values == "alternating":
        filt[:, :, :3, :3] = rng.choice([-128, 127], size=(2, 2, 3, 3))
        x[:, :7, :7] = rng.choice([-128, 127], size=(2, 7, 7))
        bias[:] = -(1 << 31), 1 << 20
    return filt, bias, x, uo


# ---- a CPU source check: no call's own shared-memory request becomes a kernel's process-wide limit -----------------------------
# kernels whose limit is set to the call's own request, and why only one request above 48 KB can reach them
SMEM_PER_CALL = {
    "k_encode_small<T>": "one request above 48 KB per element type: the whole codeword in shared memory only up to 64 KB, so only "
                         "nv = 12 (Base) or nv = 11 (Ext) asks for more than 48 KB",
    "k_tile_pass<T,MODE>": "never above 48 KB: a tile is at most 2^11 Base or 2^10 Ext values, or 2^7 rows of 2^4 columns (32 KB)",
}


def _shape_free(expr, consts, locals_):
    """True when `expr` uses only literals, sizeof(...), casts and file-scope constants (through local const definitions)"""
    expr = re.sub(r"sizeof\s*\([^()]*\)", "0", expr)
    for name in re.findall(r"[A-Za-z_]\w*", expr):
        if name in ("int", "size_t", "u32", "u64", "unsigned", "long") or name in consts:
            continue
        if name in locals_ and _shape_free(locals_[name], consts, {k: v for k, v in locals_.items() if k != name}):
            continue
        return False
    return True


def smem_limit_calls():
    """[(file, line, kernel, value, shape free)] for every cudaFuncSetAttribute(.., MaxDynamicSharedMemorySize, ..) in csrc/"""
    found = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        src = strip_comments(open(path).read())
        consts = {d.split("=")[0].strip() for decl in re.findall(r"constexpr\s+[\w:<>]+\s+([^;()]+);", src) for d in decl.split(",")}
        for m in re.finditer(r"cudaFuncSetAttribute\s*\(\s*([\w:]+(?:<[^<>]*>)?)\s*,\s*cudaFuncAttributeMaxDynamicSharedMemorySize\s*,\s*([^;]+?)\)\s*\)\s*;", src):
            kernel, value = re.sub(r"\s+", "", m.group(1)), m.group(2).strip()
            body = src[src.rfind("\n}", 0, m.start()):m.start()]           # the enclosing function up to the call
            locals_ = dict(re.findall(r"const\s+(?:int|size_t|u32|u64)\s+(\w+)\s*=\s*([^;]+);", body))
            found.append((os.path.basename(path), src.count("\n", 0, m.start()) + 1, kernel, value, _shape_free(value, consts, locals_)))
    return found


def test_shared_memory_limits_never_follow_the_call():
    """cudaFuncSetAttribute's limit is process-wide: a thread that sets it to its own smaller request can refuse another thread's
    larger launch between that thread's set and its launch.  So the limit is the largest request of any admitted shape, unless the
    kernel has only one request above 48 KB (listed with the reason)."""
    calls = smem_limit_calls()
    assert len(calls) >= 5 and any(c[2] == "k_fft_rows" for c in calls), calls
    bad = ["%s:%d %s <- %s" % c[:4] for c in calls if not c[4] and c[2] not in SMEM_PER_CALL]
    assert bad == [], "a shared-memory limit set to the call's own request:\n" + "\n".join(bad)
    assert {c[2] for c in calls if not c[4]} == set(SMEM_PER_CALL), "listed kernels whose limit no longer follows the call"


def test_shape_check_tells_the_two_apart():
    consts, locals_ = {"FFT_ROWS_MAX_LOG"}, {"smem_max": "(int)(sizeof(gle) << FFT_ROWS_MAX_LOG)", "smem": "sizeof(gle) << log_n"}
    assert _shape_free("smem_max", consts, locals_)
    assert not _shape_free("(int)smem", consts, locals_)
    assert not _shape_free("(int)(sizeof(gle) << log_n)", consts, locals_)


# ================================================ GPU: kernel by kernel ======================================================
_WARM = []


def counted(gpu, call):
    """run call() (a dp_ function returning a status), check it, and return how many kernels it launched"""
    lib = gpu.lib()
    if not _WARM:     # the power table is built on first use
        h = C.c_void_p()
        a = np.array([1, 0], dtype=np.uint64)
        gpu.check(lib.dp_phi_level(1, 1, 0, O.ptr(a), O.ptr(a), 0, C.byref(h)))
        gpu.Mle(h.value).free()
        _WARM.append(1)
    before = lib.dp_kernel_launches()
    gpu.check(call())
    return lib.dp_kernel_launches() - before


def out_mle(gpu, call):
    """(Mle, launches) for a dp_ call whose last argument is the output handle"""
    h = C.c_void_p()
    k = counted(gpu, lambda: call(C.byref(h)))
    return gpu.Mle(h.value), k


def run_fft(gpu, rows, log_n, inverse):
    m = gpu.Mle.upload(rows.reshape(-1, 2), True)
    fn = gpu.lib().dp_fft_rows if log_n <= 13 else gpu.lib().dp_fft_rows_long
    k = counted(gpu, lambda: fn(m.h, log_n, inverse))
    out = m.download().reshape(-1, 1 << log_n, 2)
    m.free()
    return out, k


def check_fft_batch(gpu, pats, log_n):
    """the rows of `pats` as one MLE, transformed forward and (from the same input) inverse: one launch for rows up to 2^13, two
    (the four-step passes) above"""
    rows = np.stack([row() for _, row, _ in pats])
    for inverse in (0, 1):
        got, k = run_fft(gpu, rows, log_n, inverse)
        assert k == (1 if log_n <= 13 else 2)
        for r, (name, _, transform) in enumerate(pats):
            assert (got[r] == transform(inverse)).all(), "%s, inverse=%d, %d rows" % (name, inverse, len(pats))


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", range(1, 14))
def test_fft_rows(gpu, log_n):
    """every pattern in one batch of rows, padded to 16 with random rows, and the random row alone"""
    pats = fft_patterns(log_n)
    check_fft_batch(gpu, pats + [random_pattern(log_n, i) for i in range(16 - len(pats))], log_n)
    check_fft_batch(gpu, [pats[-1]], log_n)


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", range(14, 22))
def test_fft_rows_long(gpu, log_n):
    """the patterns two rows at a time, and the random row alone"""
    pats = fft_patterns(log_n)
    for i in range(0, len(pats) - 1, 2):
        check_fft_batch(gpu, pats[i:i + 2], log_n)
    check_fft_batch(gpu, [pats[-1]], log_n)


def phi_device(gpu, rx, scale, n, is_fft):
    rxw, sw = u64e(list(rx)), u64e([scale])
    mids = (C.c_void_p * (n - 1))()
    fn = gpu.lib().dp_phi_g_init if n <= 14 else gpu.lib().dp_phi_g_init_long
    w, k = out_mle(gpu, lambda out: fn(O.ptr(rxw), n, O.ptr(sw), is_fft, out, mids))
    got = w.download()
    w.free()
    got_mid = []
    for h in mids:
        mm = gpu.Mle(h)
        got_mid.append(mm.download())
        mm.free()
    return got, got_mid, k


def phi_launches(n, is_fft):
    if n <= 14:
        return 1
    last = n if is_fft else n - 1
    head = min(last, 11)
    return 1 + (last - head) + (1 if not is_fft and head < last else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("n", range(2, 22))
@pytest.mark.parametrize("is_fft", [1, 0])
@pytest.mark.parametrize("case", PHI_CASES)
def test_phi_g_init(gpu, n, is_fft, case):
    """w_red and every mid table; the Python restatement up to 2^15, the same steps on the checker's field operations (pinned to it
    on the CPU) above"""
    rx, scale = phi_inputs(case, n)
    got, got_mid, k = phi_device(gpu, rx, scale, n, is_fft)
    assert k == phi_launches(n, is_fft)
    if n <= 15:
        phi_g, mid = ref_phi_g_init(rx, scale, n, is_fft)
        phi_g, mid = u64e(phi_g), [u64e(t) for t in mid]
    else:
        phi_g, mid = fast_phi_g_init(rx, scale, n, is_fft)
    assert (got == phi_g).all()
    assert len(got_mid) == n - 1
    for i, (a, b) in enumerate(zip(got_mid, mid)):
        assert (a == b).all(), "mid[%d]" % i


@pytest.mark.gpu
@pytest.mark.parametrize("n_total", list(range(1, 22)) + [32])
def test_phi_level(gpu, n_total):
    """shift 0 and the largest shift, both directions, A and B random and at the edges.  n_total = 32 is admitted by the ABI:
    there `1u << n_total` in k_phi_level is a shift by the full width"""
    len_log = min(n_total, 10)
    rnd = [tuple(map(int, e)) for e in rand_e(_seed("phi level", n_total), 2)]
    ab = [tuple(rnd), (ZERO, ONE), ((P - 1, 0), (P - 1, 0)), ((P - 1, P - 1), (P - 1, P - 1)), ((0, 1), (P - 1, 0)), (ONE, ZERO)]
    for shift in sorted({0, n_total - len_log}):
        for inverse in (0, 1):
            for A, B in ab:
                a, b = u64e([A]), u64e([B])
                m, k = out_mle(gpu, lambda out: gpu.lib().dp_phi_level(len_log, n_total, shift, O.ptr(a), O.ptr(b), inverse, out))
                got = m.download()
                m.free()
                assert k == 1
                assert (got == u64e(ref_phi_level(len_log, n_total, shift, A, B, inverse))).all(), (shift, inverse, A, B)


CONV_PROD_CASES = [(kx, kw, n, v) for kx in (1, 2, 16, 64) for kw in (1, 4) for n, v in ((1, "random"), (8, "random"), (8, "p-1"),
                                                                                      (64, "base p-1"))] \
    + [(1, 4, 1 << 16, "random"), (2, 4, 1 << 16, "p-1"), (2, 1, 1 << 18, "random")]   # kw n > 132 SMs x 8 x 128: the grid strides


@pytest.mark.gpu
@pytest.mark.parametrize("kx,kw,n,values", CONV_PROD_CASES)
def test_conv_prod(gpu, kx, kw, n, values):
    """random operands and operands at p - 1, as Ext values and as Base values lifted.  MLE lengths are powers of two, so kx and
    kw are too."""
    x, w = rand_e(_seed("x", kx, n), kx * n), rand_e(_seed("w", kw, kx, n), kw * kx * n)
    if values == "p-1":
        x[:], w[:] = P - 1, P - 1
    elif values == "base p-1":
        x[:, 0], w[:, 0], x[:, 1], w[:, 1] = P - 1, P - 1, 0, 0
        x[::3, 0] = 1
    xm, wm = gpu.Mle.upload(x, True), gpu.Mle.upload(w, True)
    m, k = out_mle(gpu, lambda out: gpu.lib().dp_conv_prod(xm.h, wm.h, kw, kx, C.c_uint64(n), out))
    assert k == 1
    assert (m.download() == ref_conv_prod(x, w, kw, kx, n)).all()
    for t in (m, xm, wm):
        t.free()


@pytest.mark.gpu
@pytest.mark.parametrize("is_ext", [True, False])
@pytest.mark.parametrize("rows,n_real,n,wide", [(1, 2, 4, False), (4, 4, 4, False), (2, 2, 8, True), (1, 8, 8, True), (2, 1, 16, False),
                                                (4, 4, 8, True), (2, 64, 512, True)])
def test_pad_rows(gpu, is_ext, rows, n_real, n, wide):
    """n_real < n and n_real = n, out_len = n^2 and 2 n^2, Base and Ext sources; the last case makes the grid stride"""
    out_len = (2 if wide else 1) * n * n
    cnt = rows * n_real * n_real
    src = rand_e(_seed("pad", rows, n_real, n), cnt) if is_ext else O.splitmix_f(_seed("pad", rows, n_real, n), cnt)
    sm = gpu.Mle.upload(src, is_ext)
    m, k = out_mle(gpu, lambda out: gpu.lib().dp_pad_rows(sm.h, C.c_uint64(rows), n_real, n, C.c_uint64(out_len), out))
    assert k == 1
    assert (m.download() == ref_pad_rows(src, rows, n_real, n, out_len)).all()
    m.free()
    sm.free()


@pytest.mark.gpu
@pytest.mark.parametrize("length,row_len", [(1, 1), (64, 1), (64, 64), (64, 8), (1 << 20, 1 << 20), (1 << 20, 1 << 7)])
def test_reverse_rows(gpu, length, row_len):
    src = O.splitmix_f(_seed("rev", length), length)
    sm = gpu.Mle.upload(src, False)
    m, k = out_mle(gpu, lambda out: gpu.lib().dp_reverse_rows(sm.h, C.c_uint64(row_len), out))
    assert k == 1
    assert (m.download() == ref_reverse_rows(src, row_len)).all()
    m.free()
    sm.free()


@pytest.mark.gpu
@pytest.mark.parametrize("length,times", [(1, 1), (1, 8), (8, 1), (8, 2), (64, 16), (1 << 16, 32)])
def test_mle_repeat(gpu, length, times):
    src = rand_e(_seed("repeat", length), length)
    sm = gpu.Mle.upload(src, True)
    m, k = out_mle(gpu, lambda out: gpu.lib().dp_mle_repeat(sm.h, times, out))
    assert k == 1
    assert (m.download() == np.tile(src, (times, 1))).all()
    m.free()
    sm.free()


def conv_rows(kw, n_x, seed):
    """[kw, 2 n_x^2] Ext rows whose c0 sweeps 0, 1, (p - 1)/2, (p + 1)/2, p - 1 and random values; c1 is random (ignored)"""
    nx2 = n_x * n_x
    rows = rand_e(seed, kw * 2 * nx2)
    edges = np.array([0, 1, HALF, HALF + 1, P - 1, HALF - 1, HALF + 2, 2], dtype=np.uint64)
    rows[::3, 0] = np.resize(edges, rows[::3, 0].shape)
    rows[1::7, 0] = np.resize(np.arange(1, 40, dtype=np.uint64), rows[1::7, 0].shape)    # small positive
    rows[2::7, 0] = np.resize(P - np.arange(1, 40, dtype=np.uint64), rows[2::7, 0].shape)  # small negative
    return rows


CONV_OUT_SHAPES = [(1, 1), (1, 2), (2, 4), (4, 8), (2, 512)]   # (kw, n_x); the last makes the grid stride
# Element is i64: to_element((p - 1)/2) + 2^31 - 1 is INT64_MAX and to_element((p + 1)/2) - 2^31 is INT64_MIN, both reached at kw = 4
BIASES = np.array([-5, 3, -(1 << 31), (1 << 31) - 1], dtype=np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("kw,n_x", CONV_OUT_SHAPES)
def test_conv_output_elements(gpu, kw, n_x):
    """to_element's (p - 1)/2 sign boundary, biases that cross zero.  The product itself does not call dp_conv_output_elements
    today (dp_conv_output keeps the output on the device), but it is part of the C ABI."""
    rows = conv_rows(kw, n_x, _seed("elements", kw, n_x))
    bias = np.array(BIASES[:kw], dtype=np.int64)
    rm = gpu.Mle.upload(rows, True)
    out = np.zeros(kw * n_x * n_x, dtype=np.int64)
    k = counted(gpu, lambda: gpu.lib().dp_conv_output_elements(rm.h, kw, n_x, O.ptr(bias), O.ptr(out)))
    assert k == 1
    assert (out == ref_conv_output_elements(rows, kw, n_x, bias)).all()
    rm.free()


@pytest.mark.gpu
@pytest.mark.parametrize("kw,n_x", CONV_OUT_SHAPES)
def test_conv_output(gpu, kw, n_x):
    """after = c0 + bias and cleared = after * mask, field words, with biases below zero and masks that clear some entries"""
    rows = conv_rows(kw, n_x, _seed("output", kw, n_x))
    bias_f = field(BIASES[:kw])
    mask = (np.arange(kw * n_x * n_x) % 3 != 1).astype(np.uint64)
    rm, bm, mm = gpu.Mle.upload(rows, True), gpu.Mle.upload(bias_f, False), gpu.Mle.upload(mask, False)
    ha, hc = C.c_void_p(), C.c_void_p()
    k = counted(gpu, lambda: gpu.lib().dp_conv_output(rm.h, kw, n_x, bm.h, mm.h, C.byref(ha), C.byref(hc)))
    after, cleared = gpu.Mle(ha.value), gpu.Mle(hc.value)
    assert k == 1
    ea, ec = ref_conv_output(rows, kw, n_x, bias_f, mask)
    assert (after.download() == ea).all()
    assert (cleared.download() == ec).all()
    for t in (after, cleared, rm, bm, mm):
        t.free()


@pytest.mark.gpu
@pytest.mark.parametrize("values", ["extreme", "alternating"])
def test_conv_layer_at_extreme_values(gpu, values):
    """-128 weights on 127 inputs, or random extremes of both signs, with biases at the ends of 32 bits: inference tensors and
    the whole flat layer proof equal the checker's"""
    filt, bias, x, uo = extreme_conv(values)
    after, cleared, got = gpu.conv_prove(filt, bias, uo, x)
    ea, ec = O.conv_op(filt, bias, uo, x)
    assert (after == ea).all() and (cleared == ec).all()
    if values == "alternating":
        assert (ea > 0).any() and (ea < 0).any()
    exp = O.conv_prove(filt, bias, uo, x)
    assert got.shape == exp.shape and (got == exp).all()


def _conv_output_call(gpu, rows_len, rows_ext, bias_len, bias_ext, mask_len):
    rows = gpu.Mle.upload(rand_e(1, rows_len) if rows_ext else O.splitmix_f(1, rows_len), rows_ext)
    bias = gpu.Mle.upload(rand_e(2, bias_len) if bias_ext else O.splitmix_f(2, bias_len), bias_ext)
    mask = gpu.Mle.upload(np.ones(mask_len, dtype=np.uint64), False)
    return gpu.lib().dp_conv_output(rows.h, 2, 4, bias.h, mask.h, C.byref(C.c_void_p()), C.byref(C.c_void_p()))   # kw 2, n_x 4


def _reverse_call(gpu, ext_src, length, row_len):
    src = gpu.Mle.upload(rand_e(3, length) if ext_src else O.splitmix_f(3, length), ext_src)
    return gpu.lib().dp_reverse_rows(src.h, C.c_uint64(row_len), C.byref(C.c_void_p()))


ROWS = "dp_conv_output: need [kw, 2 n_x^2] Ext rows"
BIAS_MASK = "dp_conv_output: need a Base bias [kw] and a Base mask [kw, n_x, n_x]"
WHOLE_ROWS = "dp_reverse_rows: need a Base MLE of whole rows"
REFUSALS = {   # case -> (call, dp_last_error text); every one returns DP_ERR_INVALID
    "conv_output rows too short": (lambda g: _conv_output_call(g, 32, True, 2, False, 32), ROWS),
    "conv_output Base rows": (lambda g: _conv_output_call(g, 64, False, 2, False, 32), ROWS),
    "conv_output Ext bias": (lambda g: _conv_output_call(g, 64, True, 2, True, 32), BIAS_MASK),
    "conv_output bias length": (lambda g: _conv_output_call(g, 64, True, 4, False, 32), BIAS_MASK),
    "conv_output mask length": (lambda g: _conv_output_call(g, 64, True, 2, False, 16), BIAS_MASK),
    "reverse_rows of an Ext MLE": (lambda g: _reverse_call(g, True, 8, 2), WHOLE_ROWS),
    "reverse_rows row_len 0": (lambda g: _reverse_call(g, False, 8, 0), WHOLE_ROWS),
    "reverse_rows partial row": (lambda g: _reverse_call(g, False, 8, 3), WHOLE_ROWS),
    "reverse_rows row longer than the MLE": (lambda g: _reverse_call(g, False, 8, 16), WHOLE_ROWS),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(REFUSALS))
def test_refusal(gpu, case):
    """each refusal returns DP_ERR_INVALID and its message, and the context it happened in still proves a layer like the checker"""
    call, text = REFUSALS[case]
    assert call(gpu) == gpu.DP_ERR_INVALID
    assert gpu.lib().dp_last_error().decode() == text
    filt, bias, x, uo = O.synthetic_conv(2, 2, 8, 4, 2, 3, 2, 7, 45, 46)
    _, _, got = gpu.conv_prove(filt, bias, uo, x)
    assert (got == O.conv_prove(filt, bias, uo, x)).all()
