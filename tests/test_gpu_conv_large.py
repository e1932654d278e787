"""Convolutions on images wider than 64 pixels on the device (csrc/conv.cu dp_fft_rows_long / dp_phi_g_init_long, the
convolution output kept in HBM) against the CPU checker: the long FFT rows, their refusals, one layer proof at rows of 2^15 and
2^17, and the covid model's spatial shape (zkml/assets/scripts/covid/covid.py, 224x224) proved from its descriptor."""
import ctypes as C

import numpy as np
import pytest

import models
import oracle_py as O

pytestmark = pytest.mark.gpu


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _out():
    return C.byref(C.c_void_p())


@pytest.mark.parametrize("log_n,rows", [(14, 4), (15, 2), (17, 4), (21, 2)])
def test_fft_rows_long(gpu, log_n, rows):
    """forward equals the checker's fft; the inverse gives the input back"""
    n = 1 << log_n
    v = O.splitmix_e(90 + log_n, rows * n).reshape(rows, n, 2)
    m = gpu.Mle.upload(v.reshape(-1, 2), True)
    gpu.check(gpu.lib().dp_fft_rows_long(m.h, log_n, 0))
    got = m.download().reshape(rows, n, 2)
    assert (got == O.fft_ext(v)).all()
    gpu.check(gpu.lib().dp_fft_rows_long(m.h, log_n, 1))
    assert (m.download().reshape(rows, n, 2) == v).all()


def test_fft_rows_long_inverse(gpu):
    """the inverse alone equals the checker's inverse fft (scaled by 1/n)"""
    log_n, rows = 16, 2
    v = O.splitmix_e(77, rows << log_n).reshape(rows, 1 << log_n, 2)
    m = gpu.Mle.upload(v.reshape(-1, 2), True)
    gpu.check(gpu.lib().dp_fft_rows_long(m.h, log_n, 1))
    assert (m.download().reshape(v.shape) == O.fft_ext(v, inverse=True)).all()


def _fft_long(gpu, ext, n_elems, log_n):
    m = gpu.Mle.upload(O.splitmix_e(700, n_elems) if ext else O.splitmix_f(700, n_elems), ext)
    return gpu.lib().dp_fft_rows_long(m.h, log_n, 0)


def _phi_long(gpu, n):
    rx, scale, mid = O.splitmix_e(680, n).reshape(-1), np.array([1, 0], dtype=np.uint64), (C.c_void_p * 24)()
    return gpu.lib().dp_phi_g_init_long(_vp(rx), n, _vp(scale), 1, _out(), mid)


LONG_ROW = "dp_fft_rows_long: row length must be 2^14..2^21 and divide the MLE length"
PHI_LONG = "dp_phi_g_init_long: need 15 <= n <= 21"
REFUSALS = {   # case -> (call, dp_last_error text); every one returns DP_ERR_INVALID
    "fft_rows_long log_n = 13": (lambda g: _fft_long(g, True, 1 << 13, 13), LONG_ROW),
    "fft_rows_long log_n = 22": (lambda g: _fft_long(g, True, 1 << 14, 22), LONG_ROW),
    "fft_rows_long of a Base MLE": (lambda g: _fft_long(g, False, 1 << 14, 14), "dp_fft_rows_long: need an Ext MLE"),
    "fft_rows_long length not a multiple of the row": (lambda g: _fft_long(g, True, 1 << 14, 15), LONG_ROW),   # half a row
    "phi_g_init_long n = 14": (lambda g: _phi_long(g, 14), PHI_LONG),
    "phi_g_init_long n = 22": (lambda g: _phi_long(g, 22), PHI_LONG),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_long_refusal(gpu, case):
    """each refusal returns DP_ERR_INVALID and its message, and the context it happened in still proves a layer like the checker"""
    call, text = REFUSALS[case]
    assert call(gpu) == gpu.DP_ERR_INVALID
    assert gpu.lib().dp_last_error().decode() == text
    filt, bias, x, uo = O.synthetic_conv(2, 2, 8, 4, 2, 3, 2, 7, 45, 46)
    _, _, got = gpu.conv_prove(filt, bias, uo, x)
    assert (got == O.conv_prove(filt, bias, uo, x)).all()


# (kw, kx, n_x, real_nw, kw_u, k_u, kx_u, n_x_u): rows of 2 n_x^2 = 2^15 and 2^17, a 3x3 filter on 110 / 222 real pixels
LARGE_SHAPES = [(4, 2, 128, 4, 3, 3, 2, 110), (2, 4, 256, 4, 2, 3, 3, 222)]


@pytest.mark.parametrize("kw,kx,n_x,rn,kw_u,k_u,kx_u,n_x_u", LARGE_SHAPES)
def test_conv_layer_large(gpu, kw, kx, n_x, rn, kw_u, k_u, kx_u, n_x_u):
    """inference tensors and the whole flat layer proof (its phi tables of 2^16 / 2^18 come from dp_phi_g_init_long)"""
    filt, bias, x, uo = O.synthetic_conv(kw, kx, n_x, rn, kw_u, k_u, kx_u, n_x_u, 55, 56)
    after, cleared, got = gpu.conv_prove(filt, bias, uo, x, cap=1 << 22)
    ea, ec = O.conv_op(filt, bias, uo, x)
    assert (after == ea).all() and (cleared == ec).all()
    exp = O.conv_prove(filt, bias, uo, x, cap=1 << 22)
    assert got.shape == exp.shape and (got == exp).all()


def _first_difference(got, exp):
    if got.shape == exp.shape and (got == exp).all():
        return None
    n = min(got.size, exp.size)
    bad = np.nonzero(got[:n] != exp[:n])[0]
    return "%d words against %d, first difference at word %d" % (got.size, exp.size, bad[0] if bad.size else n)


_COVID = {}


def covid_small():
    """the covid model at 224x224 with 4-channel convolutions and fc = 8: (desc, data, input)"""
    if not _COVID:
        d, w, x, _ = models.covid(seed=3, channels=(4, 4, 4, 4, 4), fc=8)
        _COVID.update(desc=d, data=w, x=x)
    return _COVID["desc"], _COVID["data"], _COVID["x"]


def test_covid_shape_full_proof(gpu):
    """device ModelContext.prove equals the checker bit for bit, the restated verifier accepts, and a stored trace proves again"""
    desc, data, x = covid_small()
    ctx = gpu.ModelContext(desc, data, x.size)
    try:
        got = ctx.prove(x)
        exp, _ = O.model_prove(desc, data, x)
        assert _first_difference(got, exp) is None, _first_difference(got, exp)
        assert O.model_prove_verify(desc, data, x) is None
        ctx.run_inference(x)
        assert (ctx.prove_trace(want_proof=True) == exp).all()
    finally:
        ctx.free()


def test_covid_shape_concurrent_block_mode(gpu):
    """several proofs in flight, blocking waits, resident and end to end: every proof equals the checker's"""
    desc, data, x = covid_small()
    exp, _ = O.model_prove(desc, data, x)
    before = gpu.lib().dp_get_wait_mode()
    gpu.set_wait_mode(1)
    ctx = gpu.ModelContext(desc, data, x.size)
    try:
        ctx.run_inference(x)
        for e2e in (False, True):
            _, proofs, _ = ctx.prove_concurrent_all(4, 6, stride=exp.size + 64, e2e=e2e)
            for j, p in enumerate(proofs):
                assert _first_difference(p, exp) is None, "e2e=%d job %d: %s" % (e2e, j, _first_difference(p, exp))
    finally:
        ctx.free()
        gpu.set_wait_mode(before)


def test_covid_shape_blake3(gpu):
    """the same proof under the BLAKE3 hasher and transcript"""
    desc, data, x = covid_small()
    O.set_hash_mode(1)
    gpu.set_hasher(1)
    try:
        ctx = gpu.ModelContext(desc, data, x.size)
        try:
            got = ctx.prove(x)
        finally:
            ctx.free()
        exp, _ = O.model_prove(desc, data, x)
        assert _first_difference(got, exp) is None, _first_difference(got, exp)
    finally:
        O.set_hash_mode(0)
        gpu.set_hasher(0)


def test_conv_into_conv_32x32(gpu):
    """a 32x32 CNN whose first convolution feeds the second directly (cifar-cnn.py --without-maxpool): equals the checker"""
    desc, data, x, _ = models.covid(seed=4, img=32, channels=(6, 8), fc=16, k=3)   # conv -> conv -> maxpool -> dense
    ctx = gpu.ModelContext(desc, data, x.size)
    try:
        got = ctx.prove(x)
    finally:
        ctx.free()
    exp, _ = O.model_prove(desc, data, x)
    assert _first_difference(got, exp) is None, _first_difference(got, exp)
