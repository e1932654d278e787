"""GPU tests (-m gpu) of the device-side quantised inference and lookup-witness generation (csrc/witness.cu, SURVEY.md 8f.3)
against a numpy restatement of the reference's host loops: Dense::op, Requant::op + gen_lookup_witness
(zkml/src/layers/requant.rs:208-330), Relu gen_lookup_witness (layers/activation.rs:238-323), Maxpool2D::op + compute_polys
(layers/pooling.rs:210-271,667-771), multiplicity counting (lookup/context.rs:675-737).  Bit-exact (integers)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
P = 0xFFFFFFFF00000001
QMIN, QMAX = -127, 127


def to_field(v):
    v = np.asarray(v, dtype=np.int64)
    return np.where(v < 0, (v.astype(np.int64) + np.int64(-1)).astype(np.uint64) + np.uint64((P + 1) & 0xFFFFFFFFFFFFFFFF), v.astype(np.uint64))


def test_to_field_helper():
    assert int(to_field([-1])[0]) == P - 1 and int(to_field([5])[0]) == 5 and int(to_field([-127])[0]) == P - 127


@pytest.mark.parametrize("nrows,ncols", [(16, 16), (64, 256), (1024, 1024), (8, 2)])
def test_dense(gpu, nrows, ncols):
    rng = np.random.default_rng(nrows + ncols)
    w = rng.integers(-127, 128, size=(nrows, ncols)); b = rng.integers(-127, 128, size=nrows); x = rng.integers(-127, 128, size=ncols)
    out = gpu.Witness.dense(gpu.Mle.upload(to_field(w.reshape(-1)), False), gpu.Mle.upload(to_field(b), False), gpu.Mle.upload(to_field(x), False), nrows, ncols)
    assert (out.download() == to_field(w @ x + b)).all()


@pytest.mark.parametrize("n,width", [(64, 64), (1024, 1024), (4096, 256)])
def test_requant_columns_and_multiplicities(gpu, n, width):
    rng = np.random.default_rng(n)
    lw = width.bit_length() - 1
    fp = ((lw + 24 + 7) // 8) * 8 - lw
    shift, fpm, ibits = lw + fp, 3 << (fp - 2), 2 * 7 + lw + 1
    csize = ibits + (fpm - 1).bit_length() - shift      # Requant::clamping_size
    x = rng.integers(-(1 << (ibits - 1)), (1 << (ibits - 1)) + 1, size=n)     # the clamping table covers |cin| < 2^(csize-1): |x| <= 2^(ibits-1) stays inside (0.375 * 2^csize)
    tmp = x * fpm + (1 << (shift - 1)); cl = tmp >> shift; co = np.clip(cl, QMIN, QMAX); sh = tmp & ((1 << shift) - 1)
    chunks = [(sh >> (8 * j)) & 255 for j in range(shift // 8)]
    wit = gpu.Witness([(2, 0), (3, csize)])
    cols = wit.requant(gpu.Mle.upload(to_field(x), False), shift, fpm, ibits, 1, 0)
    assert len(cols) == 2 + shift // 8
    assert (cols[0].download() == to_field(cl)).all() and (cols[1].download() == to_field(co)).all()
    for j, c in enumerate(chunks):
        assert (cols[2 + j].download() == c.astype(np.uint64)).all()
    mults, bits = wit.finish()
    assert bits == 0
    assert (mults[0].download() == np.bincount(np.concatenate(chunks), minlength=256).astype(np.uint64)).all()
    assert (mults[1].download() == np.bincount(cl + (1 << (csize - 1)), minlength=1 << csize).astype(np.uint64)).all()


def test_requant_rejects_out_of_range_inputs(gpu):
    wit = gpu.Witness([(2, 0), (3, 10)])
    wit.requant(gpu.Mle.upload(to_field(np.array([1 << 40, 0, 0, 0])), False), 16, 3 << 6, 20, 1, 0)
    _, bits = wit.finish()
    assert bits & 1          # "Could not apply requantisation, tensor element had absolute value too large"
    wit = gpu.Witness([(2, 0), (3, 10)])
    wit.requant(gpu.Mle.upload(to_field(np.array([1 << 19, 0, 0, 0])), False), 16, 3 << 6, 20, 1, 0)   # in range for the op, outside the clamping table
    _, bits = wit.finish()
    assert bits == 2


def test_relu_and_pool(gpu):
    rng = np.random.default_rng(7)
    x = rng.integers(-127, 128, size=2048)
    wit = gpu.Witness([(0, 0), (2, 0)])
    out = wit.relu(gpu.Mle.upload(to_field(x), False), 0)
    assert (out.download() == np.maximum(x, 0).astype(np.uint64)).all()
    C, H, W = 4, 16, 16
    t = rng.integers(0, 128, size=(C, H, W))
    cols = wit.pool(gpu.Mle.upload(to_field(t.reshape(-1)), False), C, H, W, 1)
    win = t.reshape(C, H // 2, 2, W // 2, 2)
    mx = win.max(axis=(2, 4))
    assert (cols[4].download() == mx.reshape(-1).astype(np.uint64)).all()
    diffs = []
    for k, (dr, dc) in enumerate([(0, 0), (1, 0), (0, 1), (1, 1)]):
        d = (mx - win[:, :, dr, :, dc]).reshape(-1); diffs.append(d)
        assert (cols[k].download() == d.astype(np.uint64)).all()
    mults, bits = wit.finish()
    assert bits == 0
    assert (mults[0].download() == np.bincount(x + 128, minlength=256).astype(np.uint64)).all()
    assert (mults[1].download() == np.bincount(np.concatenate(diffs), minlength=256).astype(np.uint64)).all()


def test_end_to_end_proof_uses_device_inference(gpu):
    """prove(x) (inference on the device from the host input vector) == prove on the stored device trace == the CPU checker's proof"""
    import oracle_py as O
    nl, width = 2, 128
    w, b, rq = O.synthetic_mlp(nl, width, 21)
    x = O.synthetic_input(width, 22)
    exp, _ = O.zkml_prove(nl, width, 21, 22)
    ctx = gpu.ZkmlContext(nl, width, w, b, rq)
    assert (ctx.prove(x) == exp).all()
    ctx.run_inference(x)
    assert (ctx.prove_trace(want_proof=True) == exp).all()


def test_model_refuses_values_outside_the_lookups(gpu):
    """the model-level refusals of the witness pass: a Dense output past 2^intermediate_bit_size refuses the requant, a ReLU input
    past its table refuses the lookup; a refused proof leaves the context able to prove the next input bit for bit"""
    import oracle_py as O
    nl, width = 2, 128
    w, b, rq = O.synthetic_mlp(nl, width, 21)
    x = O.synthetic_input(width, 22)
    bad = x * (1 << 20)
    assert np.abs(w[: width * width].reshape(width, width) @ bad + b[:width]).max() > 1 << int(rq[0][3])
    ctx = gpu.ZkmlContext(nl, width, w, b, rq)
    with pytest.raises(gpu.DpError, match="absolute value too large"):
        ctx.prove(bad)
    exp, _ = O.zkml_prove(nl, width, 21, 22)
    assert (ctx.prove(x) == exp).all()

    n = 16
    desc = np.zeros((2, 9), dtype=np.int64)
    desc[0, :3] = 0, n, n                   # Dense n x n
    desc[1, 0] = 2                          # ReLU
    data = np.concatenate([np.ones(n * n, dtype=np.int64), np.zeros(n, dtype=np.int64)])
    with pytest.raises(gpu.DpError, match="not in its table"):
        gpu.ModelContext(desc, data, n).prove(np.full(n, 100, dtype=np.int64))     # outputs 1600 > 127
