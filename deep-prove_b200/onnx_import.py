"""Import a trained float ONNX model (Gemm / MatMul / Conv / Relu / MaxPool / Flatten / Reshape-as-flatten, one chain) into the
padded quantised layout the prover takes: the (desc, data, input_len) of dph_model_context_new plus a Metadata object that
quantises float inputs and dequantises outputs.  Pure Python + numpy: the protobuf wire format is read directly.

The quantisation restates the reference's default loader (zkml/src/parser/mod.rs:71-93: load, quantise with AbsoluteMax, pad),
or, given calibration samples, its InferenceObserver (observe(); the strategy its benchmark uses with --quantization inference):
  - AbsoluteMax without a representative input (quantization/strategy.rs:190-249): the model input and the output of every node
    that has a scaling of its own use ScalingFactor::default(), i.e. [-1, 1] over [MIN, MAX] (quantization/mod.rs:155-165);
  - quantize_model (strategy.rs:251-295): each Dense / Convolution node is quantised from its input scaling and followed by the
    Requant it returns; ReLU, MaxPool and flatten keep their input's scaling;
  - Dense / Convolution quantize_from_scalings (layers/dense.rs:243-265, layers/convolution.rs:546-577): the weights at
    from_absolute_max(max |weight|, |bias|), the bias at input scale x weight scale over a 2*BIT_LEN-bit domain
    (quantization/mod.rs:197-204), and Requant::from_scaling_factors / from_multiplier (layers/requant.rs:405-447) with the
    intermediate bit size of dense.rs:415-420 or convolution.rs:362-366 (unpadded shapes: quantisation precedes padding).
All float arithmetic is np.float32, as the reference computes in f32; f32::round rounds half away from zero.  This is a
restatement: it has not been run against the Rust quantiser, and log2 / powf may differ from the platform's libm in the last
bit for some inputs.

Padding follows models.py (the same helpers): channels and image sides go to powers of two, Dense rows to max(4, p2(rows)),
and the first Dense after a flatten has its columns spread over the padded [C][n_p][n_p] grid with zeros at the garbage
positions (padding.rs pad_matrix_to_ignore_garbage)."""
import struct

import numpy as np

import models
from models import REQUANT, RELU, POOL, BIT_LEN, _p2, _clog2

# ---- protobuf wire format ----------------------------------------------------------------------------------------------

def _varint(b, i):
    r = s = 0
    while True:
        c = b[i]
        i += 1
        r |= (c & 0x7F) << s
        s += 7
        if c < 0x80:
            return r, i


def _fields(b):
    """[(field number, wire type, value)]: an int for varints, bytes for the rest"""
    out, i = [], 0
    while i < len(b):
        key, i = _varint(b, i)
        f, t = key >> 3, key & 7
        if t == 0:
            v, i = _varint(b, i)
        elif t == 1:
            v, i = b[i:i + 8], i + 8
        elif t == 5:
            v, i = b[i:i + 4], i + 4
        elif t == 2:
            n, i = _varint(b, i)
            v, i = b[i:i + n], i + n
        else:
            raise ValueError("ONNX: unsupported protobuf wire type %d" % t)
        out.append((f, t, v))
    return out


def _signed(v):
    return v - (1 << 64) if v >= 1 << 63 else v


def _ints(fs, num):
    """repeated int64 field `num`, packed or not"""
    out = []
    for f, t, v in fs:
        if f != num:
            continue
        if t == 0:
            out.append(_signed(v))
        else:
            i = 0
            while i < len(v):
                x, i = _varint(v, i)
                out.append(_signed(x))
    return out


def _str(fs, num):
    return next((v.decode() for f, _, v in fs if f == num), "")


def _tensor(b):
    """TensorProto -> (name, np array): float32 from float_data (4) or raw_data (9); int64 (data_type 7) from int64_data (7) or
    raw_data"""
    fs = _fields(b)
    dims, name = _ints(fs, 1), _str(fs, 8)
    dt = next((v for f, _, v in fs if f == 2), 1)
    raw = b"".join(v for f, _, v in fs if f == 9)
    if dt == 1:
        if raw:
            a = np.frombuffer(raw, dtype="<f4")
        else:
            vals = []
            for f, t, v in fs:
                if f == 4:
                    vals.extend(struct.unpack("<%df" % (len(v) // 4), v))
            a = np.asarray(vals, dtype=np.float32)
    elif dt == 7:
        a = np.frombuffer(raw, dtype="<i8") if raw else np.asarray(_ints(fs, 7), dtype=np.int64)
    else:
        raise ValueError("ONNX: initializer %r has data type %d; only float32 weights (and int64 shapes) are supported" % (name, dt))
    return name, a.astype(a.dtype.newbyteorder("=")).reshape(dims)


def _attrs(fs):
    """AttributeProto (name 1, f 2, i 3, ints 8) -> {name: float | int | [int]}"""
    out = {}
    for f, _, v in fs:
        if f != 5:
            continue
        af = _fields(v)
        name = _str(af, 1)
        ints = _ints(af, 8)
        if ints or any(g == 8 for g, _, _ in af):
            out[name] = ints
        elif any(g == 3 for g, _, _ in af):
            out[name] = _signed(next(x for g, _, x in af if g == 3))
        elif any(g == 2 for g, _, _ in af):
            out[name] = struct.unpack("<f", next(x for g, _, x in af if g == 2))[0]
    return out


def _value_info_shape(b):
    """ValueInfoProto (name 1, type 2) -> (name, dims); TypeProto.tensor_type 1 -> shape 2 -> dim 1 -> dim_value 1 (a symbolic
    dim_param reads as -1)"""
    fs = _fields(b)
    name, dims = _str(fs, 1), []
    for tt in (v for f, _, v in _fields(next((v for f, _, v in fs if f == 2), b"")) if f == 1):
        for sh in (v for f, _, v in _fields(tt) if f == 2):
            for d in (v for f, _, v in _fields(sh) if f == 1):
                dv = [x for f, t, x in _fields(d) if f == 1 and t == 0]
                dims.append(_signed(dv[0]) if dv else -1)
    return name, dims


def read_graph(data):
    """ModelProto bytes -> (nodes, initializers, [(input name, dims)], [output names]); nodes are dicts with op, name, inputs,
    outputs, attrs"""
    graph = next((v for f, _, v in _fields(data) if f == 7), None)
    if graph is None:
        raise ValueError("ONNX: the model has no graph")
    nodes, inits, inputs, outputs = [], {}, [], []
    for f, _, v in _fields(graph):
        if f == 1:
            nf = _fields(v)
            nodes.append({"inputs": [x.decode() for g, _, x in nf if g == 1], "outputs": [x.decode() for g, _, x in nf if g == 2],
                          "name": _str(nf, 3), "op": _str(nf, 4), "attrs": _attrs(nf)})
        elif f == 5:
            name, a = _tensor(v)
            inits[name] = a
        elif f == 11:
            inputs.append(_value_info_shape(v))
        elif f == 12:
            outputs.append(_value_info_shape(v)[0])
    return nodes, inits, [i for i in inputs if i[0] not in inits], outputs


# ---- float model: one chain of supported layers -----------------------------------------------------------------------------

class FloatModel:
    """input_shape: (n,) or (C, H, W) without the batch dimension; layers: ("dense", W [out, in], b [out]), ("conv", F [o, i, k, k],
    b [o]), ("relu",), ("maxpool",), ("flatten",) -- float32"""

    def __init__(self, input_shape, layers):
        self.input_shape, self.layers = tuple(input_shape), layers

    def ops(self):
        return [l[0] for l in self.layers]

    def forward(self, x):
        """float inference in numpy (float64 accumulation of the float32 weights) on one unpadded input"""
        y = np.asarray(x, dtype=np.float64)
        for y in self.outputs(x):
            pass
        return y.reshape(-1)

    def outputs(self, x):
        """the float inference of forward(), yielding each layer's output in its unpadded shape"""
        x = np.asarray(x, dtype=np.float64).reshape(self.input_shape)
        for l in self.layers:
            if l[0] == "dense":
                x = l[1].astype(np.float64) @ x.reshape(-1) + l[2]
            elif l[0] == "conv":
                f = l[1].astype(np.float64)
                k = f.shape[2]
                h, w = x.shape[1] - k + 1, x.shape[2] - k + 1
                win = np.lib.stride_tricks.sliding_window_view(x, (k, k), axis=(1, 2))[:, :h, :w]   # [i, h, w, k, k]
                x = np.einsum("ihwab,oiab->ohw", win, f) + l[2][:, None, None]
            elif l[0] == "relu":
                x = np.maximum(x, 0)
            elif l[0] == "maxpool":
                c, h, w = x.shape
                x = x[:, :h // 2 * 2, :w // 2 * 2].reshape(c, h // 2, 2, w // 2, 2).max(axis=(2, 4))
            else:
                x = x.reshape(-1)
            yield x


def _node_label(n):
    return "%s node %r" % (n["op"], n["name"] or (n["outputs"][0] if n["outputs"] else "?"))


def _refuse(n, why):
    raise ValueError("ONNX: %s: %s" % (_node_label(n), why))


def _weight(n, inits, name):
    if name not in inits:
        _refuse(n, "input %r is not a constant initializer" % name)
    return inits[name].astype(np.float32)


def load_float(data):
    """ONNX bytes -> FloatModel.  Refuses, naming the op and the node: any op other than Gemm / MatMul / Conv / Relu / MaxPool /
    Flatten / Reshape (as a flatten) -- the ones the reference's loader registers (parser/onnx.rs:147-157); a Conv with pads,
    strides, dilations or group other than 0 / 1 / 1 / 1 (parser/onnx.rs:648-698); a MaxPool other than 2x2 with stride 2; and a
    graph that is not one chain from the input to the output."""
    nodes, inits, inputs, outputs = read_graph(data)
    if len(inputs) != 1 or len(outputs) != 1:
        raise ValueError("ONNX: the graph must have exactly one input and one output (has %d and %d)" % (len(inputs), len(outputs)))
    in_name, dims = inputs[0]
    if len(dims) in (2, 4):
        if dims[0] not in (1, -1):
            raise ValueError("ONNX: input %r has batch dimension %d; only one input at a time is supported" % (in_name, dims[0]))
        dims = dims[1:]
    if len(dims) not in (1, 3) or any(d <= 0 for d in dims):
        raise ValueError("ONNX: input %r has shape %s; a vector [n] or an image [C, H, W] (after the batch) is supported" % (in_name, dims))
    cur, layers = in_name, []
    for n in nodes:
        op, a = n["op"], n["attrs"]
        data_in = [x for x in n["inputs"] if x and x not in inits]
        if data_in != [cur] or len(n["outputs"]) != 1:
            _refuse(n, "the graph is not a single chain (the node's non-constant inputs are %s, expected [%r])" % (data_in, cur))
        if n["inputs"][0] != cur:
            _refuse(n, "the data input must be the first input")
        if op == "Gemm":
            if a.get("transA", 0) != 0 or a.get("alpha", 1.0) != 1.0 or a.get("beta", 1.0) != 1.0:
                _refuse(n, "only transA = 0, alpha = 1, beta = 1 is supported")
            w = _weight(n, inits, n["inputs"][1])
            w = w if a.get("transB", 0) else w.T
            b = _weight(n, inits, n["inputs"][2]).reshape(-1) if len(n["inputs"]) > 2 and n["inputs"][2] else np.zeros(w.shape[0], np.float32)
            if w.ndim != 2 or b.shape != (w.shape[0],):
                _refuse(n, "weight %s and bias %s are not a [out, in] matrix and an [out] vector" % (w.shape, b.shape))
            layers.append(("dense", np.ascontiguousarray(w), b))
        elif op == "MatMul":                                  # x @ B with B [in, out]: a dense layer without bias
            w = _weight(n, inits, n["inputs"][1])
            if w.ndim != 2:
                _refuse(n, "the constant operand must be a matrix, it has shape %s" % (w.shape,))
            layers.append(("dense", np.ascontiguousarray(w.T), np.zeros(w.shape[1], np.float32)))
        elif op == "Conv":
            f = _weight(n, inits, n["inputs"][1])
            k = f.shape[2] if f.ndim == 4 else 0
            for attr, ok in (("pads", 0), ("strides", 1), ("dilations", 1)):
                if any(v != ok for v in a.get(attr, [ok])):
                    _refuse(n, "%s = %s is not supported (only %s = %d)" % (attr, a[attr], attr, ok))
            if a.get("group", 1) != 1:
                _refuse(n, "group = %d is not supported (only group = 1)" % a["group"])
            if a.get("auto_pad", "NOTSET") not in ("NOTSET", "VALID"):
                _refuse(n, "auto_pad is not supported")
            if f.ndim != 4 or f.shape[3] != k or k < 2 or a.get("kernel_shape", [k, k]) != [k, k]:
                _refuse(n, "only square 2-D kernels larger than 1x1 are supported (filter %s)" % (f.shape,))
            b = _weight(n, inits, n["inputs"][2]).reshape(-1) if len(n["inputs"]) > 2 and n["inputs"][2] else np.zeros(f.shape[0], np.float32)
            layers.append(("conv", f, b))
        elif op == "MaxPool":
            if (a.get("kernel_shape") != [2, 2] or a.get("strides", [1, 1]) != [2, 2] or any(v != 0 for v in a.get("pads", [0]))
                    or any(v != 1 for v in a.get("dilations", [1])) or a.get("ceil_mode", 0) != 0):
                _refuse(n, "only a 2x2 kernel with stride 2, no padding, dilation 1 and ceil_mode 0 is supported")
            layers.append(("maxpool",))
        elif op == "Relu":
            layers.append(("relu",))
        elif op == "Flatten":
            if a.get("axis", 1) != 1:
                _refuse(n, "only axis = 1 is supported")
            layers.append(("flatten",))
        elif op == "Reshape":
            shape = inits.get(n["inputs"][1]) if len(n["inputs"]) > 1 else None
            if shape is None or not (shape.size == 1 or (shape.size == 2 and shape.reshape(-1)[0] == 1)):
                _refuse(n, "only a reshape to [-1] or [1, -1] (a flatten) is supported")
            layers.append(("flatten",))
        else:
            _refuse(n, "unsupported op %r (supported: Gemm, MatMul, Conv, Relu, MaxPool, Flatten, Reshape as flatten)" % op)
        cur = n["outputs"][0]
    if cur != outputs[0]:
        raise ValueError("ONNX: the graph is not a single chain: its output %r is not the last node's output %r" % (outputs[0], cur))
    m = FloatModel(dims, layers)
    _check_shapes(m)
    return m


def _check_shapes(m):
    """walk the unpadded shapes; refuse what the padded layout cannot hold"""
    shape = m.input_shape
    if len(shape) == 3 and shape[1] != shape[2]:
        raise ValueError("ONNX: input image %s is not square; the padded layout holds [C, n, n] images" % (shape,))
    for i, l in enumerate(m.layers):
        if l[0] == "dense":
            n_in = int(np.prod(shape))
            if len(shape) != 1 or l[1].shape[1] != n_in:
                raise ValueError("ONNX: layer %d (dense %s) does not fit its input of shape %s" % (i, l[1].shape, shape))
            shape = (l[1].shape[0],)
        elif l[0] == "conv":
            if len(shape) != 3 or l[1].shape[1] != shape[0] or l[1].shape[2] > shape[1]:
                raise ValueError("ONNX: layer %d (conv %s) does not fit its input of shape %s" % (i, l[1].shape, shape))
            shape = (l[1].shape[0], shape[1] - l[1].shape[2] + 1, shape[2] - l[1].shape[2] + 1)
        elif l[0] == "maxpool":
            if len(shape) != 3:
                raise ValueError("ONNX: layer %d (maxpool) needs an image input, it gets %s" % (i, shape))
            shape = (shape[0], shape[1] // 2, shape[2] // 2)
        elif l[0] == "flatten":
            shape = (int(np.prod(shape)),)
    return shape


# ---- quantisation (quantization/mod.rs ScalingFactor, restated in f32) ------------------------------------------------------

Q_MIN, Q_MAX = -(1 << (BIT_LEN - 1)) + 1, (1 << (BIT_LEN - 1)) - 1           # quantization/mod.rs:28-29
BIAS_MIN, BIAS_MAX = -(1 << (2 * BIT_LEN - 1)) + 1, (1 << (2 * BIT_LEN - 1)) - 1   # mod.rs:197-204
FIXED_POINT_SCALE = 25                                                       # layers/requant.rs:48
F32 = np.float32


def _round(x):
    """f32::round: half away from zero (exact: |x| + 0.5 is computed in float64)"""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    return (np.sign(x) * np.floor(np.abs(x) + 0.5)).astype(np.int64)


class ScalingFactor:
    """quantization/mod.rs:39-165: only the scale and the quantised domain matter to quantise and dequantise"""

    def __init__(self, scale, domain=(Q_MIN, Q_MAX)):
        self.scale, self.domain = F32(scale), domain

    @staticmethod
    def default():
        return ScalingFactor(F32(2.0) / F32(Q_MAX - Q_MIN))

    @staticmethod
    def from_absolute_max(abs_max, domain=(Q_MIN, Q_MAX)):
        a = np.abs(F32(abs_max))
        return ScalingFactor((a - (-a)) / F32(domain[1] - domain[0]), domain)

    def quantize(self, v):
        return np.clip(_round(np.asarray(v, dtype=np.float32) / self.scale), self.domain[0], self.domain[1])

    def dequantize(self, q):
        return np.asarray(q, dtype=np.int64).astype(np.float32) * self.scale

    def m(self, s2, s3):
        return self.scale * s2.scale / s3.scale


def requant_from_multiplier(multiplier, intermediate_bit_size):
    """Requant::from_multiplier (layers/requant.rs:409-435) -> (right_shift, fp_scale, fixed_point_multiplier)"""
    log_m = np.log2(F32(multiplier))
    int_part = int(abs(np.trunc(log_m)))
    epsilon = np.power(F32(2.0), F32(log_m - np.trunc(log_m)))
    fp_scale = -(-(int_part + FIXED_POINT_SCALE) // BIT_LEN) * BIT_LEN - int_part
    fpm = int(_round(epsilon * F32(1 << fp_scale)))
    if intermediate_bit_size + fp_scale > 63:
        raise ValueError("requant: intermediate bit size %d + fp scale %d exceeds 63" % (intermediate_bit_size, fp_scale))
    return int_part, fp_scale, fpm


class Metadata:
    """ModelMetadata (quantization/metadata.rs) of an imported model plus its padded IO layout"""

    def __init__(self, input_scaling, output_scaling, input_shape, padded_input_shape, output_len, padded_output_len):
        self.input_scaling, self.output_scaling = input_scaling, output_scaling
        self.input_shape, self.padded_input_shape = tuple(input_shape), tuple(padded_input_shape)
        self.output_len, self.padded_output_len = int(output_len), int(padded_output_len)

    def quantize_input(self, x):
        """inputs.rs:35-71: every value must lie in [-1, 1]; scale, round, clamp to [MIN, MAX]; then place the [input_shape] result in
        the padded layout (zeros elsewhere).  x: [*input_shape] or [n, *input_shape] -> int64 [padded length] or [n, padded length]"""
        x = np.asarray(x, dtype=np.float32)
        one = x.shape == self.input_shape
        xs = x.reshape((-1,) + self.input_shape) if x.size and (one or x.shape[1:] == self.input_shape) else None
        if xs is None:
            raise ValueError("quantize_input: expected shape %s or [n, %s], got %s" % (self.input_shape, self.input_shape, x.shape))
        if not np.all((xs >= -1.0) & (xs <= 1.0)):
            raise ValueError("quantize_input: input values must lie in [-1, 1] (the reference's QUANTIZATION_RANGE)")
        q = np.zeros((xs.shape[0],) + self.padded_input_shape, dtype=np.int64)
        q[(slice(None),) + tuple(slice(0, d) for d in self.input_shape)] = self.input_scaling.quantize(xs)
        q = q.reshape(xs.shape[0], -1)
        return q[0] if one else q

    def dequantize_output(self, y):
        """the real (unpadded) output entries, dequantised with the output scaling: [padded_output_len] or [n, padded_output_len]"""
        y = np.asarray(y, dtype=np.int64)
        if y.shape[-1] != self.padded_output_len:
            raise ValueError("dequantize_output: expected %d entries per output, got %d" % (self.padded_output_len, y.shape[-1]))
        return self.output_scaling.dequantize(y[..., :self.output_len])


class QuantizedLayer:
    """one quantised layer before padding, for inspection and for the unpadded integer inference the tests run: kind "dense" / "conv"
    with w, b (int64), rq = (right_shift, fp_scale, fixed_point_multiplier, intermediate_bit_size) of the Requant after it and
    out_sf, the ScalingFactor of the layer's output that the Requant targets"""

    def __init__(self, kind, w=None, b=None, rq=None, out_sf=None):
        self.kind, self.w, self.b, self.rq, self.out_sf = kind, w, b, rq, out_sf


def observe(fm, samples):
    """InferenceObserver::new_with_representative_input (quantization/strategy.rs:72-146): run the float model on every sample and
    take the input's and each node's output minimum and maximum over all samples (InferenceTracker, strategy.rs:148-187: plain
    min / max as f32, the percentile lines there are commented out); each scaling is from_absolute_max(max(|min|, |max|)).
    samples: [n, *input_shape] in [-1, 1] of the unpadded model, which is what the reference observes: it quantises before it
    pads (parser/mod.rs:89-90).  -> (input scaling, [output scaling of each Dense / Conv layer, None for the others]).  The float
    inference is forward()'s, in float64; only the extremes are rounded to f32."""
    x = np.asarray(samples, dtype=np.float32)
    if x.size == 0:
        raise ValueError("calibration: no samples; the reference then draws 10 inputs from its own RNG, which is not reproduced here")
    if x.shape[1:] != fm.input_shape:
        raise ValueError("calibration: expected samples of shape [n, %s], got %s"
                         % (", ".join(map(str, fm.input_shape)), list(x.shape)))
    if not np.all((x >= -1.0) & (x <= 1.0)):
        raise ValueError("calibration: sample values must lie in [-1, 1] (the reference's QUANTIZATION_RANGE)")
    lo = np.full(len(fm.layers) + 1, np.inf)
    hi = -lo
    for s in x:
        for i, y in enumerate([s] + list(fm.outputs(s))):
            lo[i], hi[i] = min(lo[i], y.min()), max(hi[i], y.max())
    sfs = []
    for i, (a, b) in enumerate(zip(lo, hi)):
        if i > 0 and fm.layers[i - 1][0] not in ("dense", "conv"):
            sfs.append(None)                      # Relu, MaxPool and flatten keep their input's scaling: theirs is not used
            continue
        m = max(abs(F32(a)), abs(F32(b)))
        if m == 0:
            raise ValueError("calibration: %s is zero on every sample, which gives a zero scaling factor"
                             % ("the input" if i == 0 else "the output of layer %d (%s)" % (i - 1, fm.layers[i - 1][0])))
        sfs.append(ScalingFactor.from_absolute_max(m))
    return sfs[0], sfs[1:]


def quantize(fm, calibration=None):
    """-> (list of QuantizedLayer with the requants, input scaling, output scaling).  Without calibration: AbsoluteMax without a
    representative input.  With calibration samples ([n, *input_shape]): InferenceObserver (observe()); each Dense / Conv requant
    targets that layer's own observed output scaling, taken before any Relu (layers/dense.rs:243-285, layers/convolution.rs:579-597),
    and Relu, MaxPool and flatten keep their input's scaling (layers/mod.rs:729-747)."""
    if calibration is None:
        in_sf, layer_sf = ScalingFactor.default(), [ScalingFactor.default()] * len(fm.layers)
    else:
        in_sf, layer_sf = observe(fm, calibration)
    sf = in_sf
    out = []
    for l, out_sf in zip(fm.layers, layer_sf):
        if l[0] in ("dense", "conv"):
            w, b = l[1], l[2]
            model_sf = ScalingFactor.from_absolute_max(max(np.abs(w).max(initial=F32(0)), np.abs(b).max(initial=F32(0))))
            bias_sf = ScalingFactor(sf.scale * model_sf.scale, (BIAS_MIN, BIAS_MAX))
            if l[0] == "dense":
                bits = 2 * (BIT_LEN - 1) + _clog2(w.shape[1]) + 1                                      # dense.rs:415-420
            else:
                bits = 2 * (BIT_LEN - 1) + _clog2(w.shape[1] * w.shape[2] * w.shape[3] + 1)            # convolution.rs:362-366
            rq = requant_from_multiplier(sf.m(model_sf, out_sf), bits) + (bits,)
            out.append(QuantizedLayer(l[0], model_sf.quantize(w), bias_sf.quantize(b), rq, out_sf))
            sf = out_sf
        else:
            out.append(QuantizedLayer(l[0]))
    return out, in_sf, sf


def pad(fm, qlayers):
    """the padded (desc [n_nodes, 9], data, input_len, padded input shape, padded output length)"""
    desc, data = [], []
    shape = fm.input_shape
    if len(shape) == 3:
        c_u, n_u, n_p = shape[0], shape[1], _p2(shape[1])
        padded_in = (_p2(c_u), n_p, n_p)
    else:
        padded_in = (_p2(shape[0]),)
    cols, real = padded_in[0], np.arange(padded_in[0]) < shape[0]      # a vector's padded length and its real entries
    flat_len = None
    for q in qlayers:
        if q.kind == "conv":
            row, filt, bias, h_out = models.conv_layer(q.w, q.b, n_p, n_u)
            desc.append(row)
            data += [filt.reshape(-1), bias]
            c_u, n_u = q.w.shape[0], h_out
        elif q.kind == "dense":
            if flat_len is not None:
                cols, real, flat_len = flat_len, flatten_real, None
            nrows = max(4, _p2(q.w.shape[0]))
            row, w, b = models.dense_layer(q.w, q.b, real, nrows)
            desc.append(row)
            data += [w.reshape(-1), b]
            cols, real = nrows, np.arange(nrows) < q.w.shape[0]
        elif q.kind == "relu":
            desc.append([RELU] + [0] * 8)
        elif q.kind == "maxpool":
            desc.append([POOL, _p2(c_u), n_p, n_p, 0, 0, 0, 0, 0])
            n_u, n_p = n_u // 2, n_p // 2
        elif q.kind == "flatten":
            if flat_len is None and len(shape) == 3:
                flatten_real, flat_len = models.flatten_mask(c_u, n_u, n_p), _p2(c_u) * n_p * n_p
                shape = (int(flatten_real.sum()),)
        if q.rq is not None:
            desc.append([REQUANT, q.rq[0], q.rq[1], q.rq[2], q.rq[3], 0, 0, 0, 0])
    if flat_len is not None:
        raise ValueError("ONNX: a flatten must be followed by a dense layer")
    return np.asarray(desc, dtype=np.int64), np.concatenate(data).astype(np.int64), int(np.prod(padded_in)), padded_in, cols


def import_onnx(path_or_bytes, calibration=None):
    """-> (desc, data, input_len, Metadata, FloatModel, quantised layers).  calibration: None for AbsoluteMax without a
    representative input (the reference's default loader), or float samples [n, *input_shape] in [-1, 1] to quantise with the
    InferenceObserver on them (quantize()); Metadata then carries the calibrated input and output scalings."""
    raw = path_or_bytes if isinstance(path_or_bytes, (bytes, bytearray)) else open(path_or_bytes, "rb").read()
    fm = load_float(bytes(raw))
    if not [l for l in fm.layers if l[0] != "relu"] or [l for l in fm.layers if l[0] != "relu"][-1][0] != "dense":
        raise ValueError("ONNX: the model must end in a dense layer (Gemm / MatMul), optionally followed by Relu")
    qlayers, in_sf, out_sf = quantize(fm, calibration)
    desc, data, input_len, padded_in, padded_out = pad(fm, qlayers)
    md = Metadata(in_sf, out_sf, fm.input_shape, padded_in, _check_shapes(fm)[0], padded_out)
    return desc, data, input_len, md, fm, qlayers
