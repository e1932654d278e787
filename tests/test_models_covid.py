"""CPU test: models.covid() mirrors zkml/assets/scripts/covid/covid.py (CNNModel) in the padded layout: its real-parameter count
and the padded shapes of its layers."""
import numpy as np

import models


def test_covid_shapes_and_parameter_count():
    desc, data, x, n_params = models.covid()
    assert n_params == 1_457_537
    assert x.size == 4 * 256 * 256
    convs = [r for r in desc if r[0] == models.CONV]
    # (kw, kx, padded input width, padded filter width, real output channels, real output height, width)
    assert [tuple(int(v) for v in r[1:8]) for r in convs] == [(32, 4, 256, 4, 32, 222, 222), (64, 32, 256, 4, 64, 220, 220),
                                                              (64, 64, 128, 4, 64, 108, 108), (128, 64, 64, 4, 128, 52, 52),
                                                              (128, 128, 32, 4, 128, 24, 24)]
    assert [2 * int(r[3]) ** 2 for r in convs] == [1 << 17, 1 << 17, 1 << 15, 1 << 13, 1 << 11]   # FFT row lengths
    kinds = [int(r[0]) for r in desc]
    C, R, A, P, D = models.CONV, models.REQUANT, models.RELU, models.POOL, models.DENSE
    assert kinds == [C, R, A, C, R, A, P] + [C, R, A, P] * 3 + [D, R, A, D, R, A]
    dense = [r for r in desc if r[0] == models.DENSE]
    assert [(int(r[1]), int(r[2])) for r in dense] == [(64, 128 * 16 * 16), (4, 64)]   # the one-output layer padded to 4 rows
    # weights in node order: filters and biases, then the dense matrices and biases
    sizes = [int(r[1] * r[2] * r[4] * r[4] + r[1]) for r in convs] + [int(r[1] * r[2] + r[1]) for r in dense]
    assert data.size == sum(sizes)
    w1 = data[sum(sizes[:5]):sum(sizes[:5]) + 64 * 32768].reshape(64, 128, 16, 16)
    assert np.count_nonzero(w1[:, :, 12:, :]) == 0 and np.count_nonzero(w1[:, :, :, 12:]) == 0   # 18,432 of 32,768 columns are real
    w2 = data[sum(sizes[:6]):sum(sizes[:6]) + 4 * 64].reshape(4, 64)
    assert np.count_nonzero(w2[1:]) == 0 and np.count_nonzero(data[sum(sizes) - 3:]) == 0
