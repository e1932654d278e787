"""FFT-convolution layer on the device (csrc/conv.cu + host/conv.hpp) against the CPU checker: inference tensors and the
whole layer proof (clearing hadamard, batch iFFT/FFT with matrix delegation, hadamard product, FFT of the weights), same
transcript -> identical flat proof (convolution.rs:697-1077)."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O

pytestmark = pytest.mark.gpu

SHAPES = [(2, 2, 8, 4, 2, 3, 2, 7), (4, 2, 8, 2, 3, 2, 2, 8), (2, 4, 16, 8, 2, 5, 3, 14), (1, 2, 8, 4, 1, 3, 2, 8), (1, 1, 8, 4, 1, 3, 1, 8),
          (16, 4, 32, 8, 12, 5, 3, 32), (64, 16, 16, 8, 33, 5, 12, 14)]   # the last two are CNN-264k's conv1 / conv2 after padding


@pytest.mark.parametrize("n,log_n", [(8, 3), (64, 6), (2048, 11), (8192, 13)])
def test_fft_rows(gpu, n, log_n):
    rows = 3 if n < 8192 else 2
    rows_p2 = 4 if rows == 3 else 2
    v = O.splitmix_e(40 + log_n, rows_p2 * n).reshape(rows_p2, n, 2)
    m = gpu.Mle.upload(v.reshape(-1, 2), True)
    gpu.check(gpu.lib().dp_fft_rows(m.h, log_n, 0))
    got = m.download().reshape(rows_p2, n, 2)
    assert (got == O.fft_ext(v)).all()
    gpu.check(gpu.lib().dp_fft_rows(m.h, log_n, 1))
    assert (m.download().reshape(rows_p2, n, 2) == v).all()


@pytest.mark.parametrize("kw,kx,n_x,rn,kw_u,k_u,kx_u,n_x_u", SHAPES)
def test_conv_inference(gpu, kw, kx, n_x, rn, kw_u, k_u, kx_u, n_x_u):
    filt, bias, x, uo = O.synthetic_conv(kw, kx, n_x, rn, kw_u, k_u, kx_u, n_x_u, 25, 26)
    after, cleared, _ = gpu.conv_prove(filt, bias, uo, x, prove=False)
    ea, ec = O.conv_op(filt, bias, uo, x)
    assert (after == ea).all() and (cleared == ec).all()


@pytest.mark.parametrize("kw,kx,n_x,rn,kw_u,k_u,kx_u,n_x_u", SHAPES)
def test_conv_layer_proof(gpu, kw, kx, n_x, rn, kw_u, k_u, kx_u, n_x_u):
    filt, bias, x, uo = O.synthetic_conv(kw, kx, n_x, rn, kw_u, k_u, kx_u, n_x_u, 35, 36)
    _, _, got = gpu.conv_prove(filt, bias, uo, x)
    exp = O.conv_prove(filt, bias, uo, x)
    assert got.shape == exp.shape
    assert (got == exp).all()


def _mle(gpu, n, ext):
    return gpu.Mle.upload(O.splitmix_e(670 + n, n) if ext else O.splitmix_f(670 + n, n), ext)


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _out():
    return C.byref(C.c_void_p())


def _fft_rows(gpu, ext, log_n):
    m = _mle(gpu, 8, ext)
    return gpu.lib().dp_fft_rows(m.h, log_n, 0)


def _pad_rows(gpu, src_len, n_real, n, out_len):
    m = _mle(gpu, src_len, True)
    return gpu.lib().dp_pad_rows(m.h, C.c_uint64(1), n_real, n, C.c_uint64(out_len), _out())


def _conv_prod(gpu, x_ext, x_len):
    x, w = _mle(gpu, x_len, x_ext), _mle(gpu, 8, True)
    return gpu.lib().dp_conv_prod(x.h, w.h, 1, 1, C.c_uint64(8), _out())


def _conv_output_elements(gpu):
    rows, bias, out = _mle(gpu, 8, True), np.zeros(1, dtype=np.int64), np.zeros(32, dtype=np.int64)
    return gpu.lib().dp_conv_output_elements(rows.h, 1, 4, _vp(bias), _vp(out))   # [1, 2 * 4^2] rows wanted, 8 given


def _phi_g_init(gpu, n):
    rx, scale, mid = O.splitmix_e(680, n).reshape(-1), np.array([1, 0], dtype=np.uint64), (C.c_void_p * 16)()
    return gpu.lib().dp_phi_g_init(_vp(rx), n, _vp(scale), 1, _out(), mid)


def _phi_level(gpu):
    a, b = np.array([1, 0], dtype=np.uint64), np.array([2, 0], dtype=np.uint64)
    return gpu.lib().dp_phi_level(3, 4, 2, _vp(a), _vp(b), 0, _out())


def _repeat(gpu, ext, times):
    m = _mle(gpu, 8, ext)
    return gpu.lib().dp_mle_repeat(m.h, times, _out())


ROW_LEN = "dp_fft_rows: row length must be 2^1..2^13 and divide the MLE length"
REFUSALS = {   # case -> (call, dp_last_error text); every one returns DP_ERR_INVALID
    "fft_rows of a Base MLE": (lambda g: _fft_rows(g, False, 3), "dp_fft_rows: need an Ext MLE"),
    "fft_rows log_n = 0": (lambda g: _fft_rows(g, True, 0), ROW_LEN),
    "fft_rows log_n = 14": (lambda g: _fft_rows(g, True, 14), ROW_LEN),
    "pad_rows n_real > n": (lambda g: _pad_rows(g, 16, 4, 2, 16), "dp_pad_rows: bad arguments"),
    "pad_rows wrong source length": (lambda g: _pad_rows(g, 8, 2, 4, 16), "dp_pad_rows: source length != rows * n_real^2"),
    "pad_rows length not a power of two": (lambda g: _pad_rows(g, 4, 2, 4, 12), "dp_pad_rows: rows * out_len must be a power of two"),
    "conv_prod with a Base operand": (lambda g: _conv_prod(g, False, 8), "dp_conv_prod: need Ext operands"),
    "conv_prod shape mismatch": (lambda g: _conv_prod(g, True, 4), "dp_conv_prod: operand shapes do not match [kx, n] / [kw, kx, n]"),
    "conv_output_elements wrong length": (_conv_output_elements, "dp_conv_output_elements: need [kw, 2 n_x^2] Ext rows"),
    "phi_g_init n = 1": (lambda g: _phi_g_init(g, 1), "dp_phi_g_init: need 2 <= n <= 14"),
    "phi_g_init n = 15": (lambda g: _phi_g_init(g, 15), "dp_phi_g_init: need 2 <= n <= 14"),
    "phi_level len_log + shift > n_total": (_phi_level, "dp_phi_level: bad arguments"),
    "repeat a Base MLE": (lambda g: _repeat(g, False, 2), "dp_mle_repeat: need an Ext MLE and a power-of-two count"),
    "repeat 3 times": (lambda g: _repeat(g, True, 3), "dp_mle_repeat: need an Ext MLE and a power-of-two count"),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_abi_refusal(gpu, case):
    """each refusal returns DP_ERR_INVALID and its message, and the context it happened in still proves a layer like the oracle"""
    call, text = REFUSALS[case]
    assert call(gpu) == gpu.DP_ERR_INVALID
    assert gpu.lib().dp_last_error().decode() == text
    filt, bias, x, uo = O.synthetic_conv(*SHAPES[0], 45, 46)
    _, _, got = gpu.conv_prove(filt, bias, uo, x)
    assert (got == O.conv_prove(filt, bias, uo, x)).all()
