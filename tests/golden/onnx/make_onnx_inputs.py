#!/usr/bin/env python3
"""Regenerates tests/golden/onnx/{mlp-iris-01,cnn-cifar-01}-inputs.npz: the calibration and evaluation samples the reference ships
beside the two models (zkml/assets/scripts/MLP/input.json.zst and CNN/input.json.zst of a deep-prove checkout).

Each .npz holds `inputs`, float32 [30, *input shape] (the JSON's flat input_data reshaped to the model's unpadded input), and
`labels`, int64 [30], the argmax of the one-hot output_data.  The JSON's pytorch_output field is not kept: it was not produced by
these .onnx files (its argmax agrees with their float forward on about half the samples), so it is no check of anything.
The .zst files are decompressed with the system libzstd through ctypes.  Run once, from anywhere:
    python tests/golden/onnx/make_onnx_inputs.py <deep-prove checkout>/zkml/assets/scripts
"""
import ctypes
import ctypes.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
MODELS = [("MLP", "mlp-iris-01", (4,)), ("CNN", "cnn-cifar-01", (3, 32, 32))]


def zstd_decompress(b):
    lib = ctypes.util.find_library("zstd")
    if lib is None:
        raise SystemExit("libzstd not found")
    z = ctypes.CDLL(lib)
    z.ZSTD_getFrameContentSize.restype = ctypes.c_ulonglong
    z.ZSTD_getFrameContentSize.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
    z.ZSTD_decompress.restype = ctypes.c_size_t
    z.ZSTD_decompress.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t]
    z.ZSTD_isError.argtypes = [ctypes.c_size_t]
    n = z.ZSTD_getFrameContentSize(b, len(b))
    if n >= 1 << 62:                          # ZSTD_CONTENTSIZE_UNKNOWN / _ERROR
        raise SystemExit("the zstd frame does not record its content size")
    out = ctypes.create_string_buffer(n)
    r = z.ZSTD_decompress(out, n, b, len(b))
    if z.ZSTD_isError(r) or r != n:
        raise SystemExit("zstd decompression failed")
    return out.raw


def main(scripts):
    for sub, name, shape in MODELS:
        with open(os.path.join(scripts, sub, "input.json.zst"), "rb") as f:
            d = json.loads(zstd_decompress(f.read()))
        x64 = np.asarray(d["input_data"], dtype=np.float64)
        x = x64.astype(np.float32)
        assert np.array_equal(x.astype(np.float64), x64), "an input value is not an f32 value"
        x = x.reshape((-1,) + shape)
        labels = np.argmax(np.asarray(d["output_data"], dtype=np.float64), axis=1).astype(np.int64)
        assert x.shape[0] == labels.shape[0] and np.all(np.abs(x) <= 1.0)
        out = os.path.join(HERE, name + "-inputs.npz")
        np.savez_compressed(out, inputs=x, labels=labels)
        print("%s: inputs %s, labels %s" % (out, x.shape, np.bincount(labels).tolist()))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
