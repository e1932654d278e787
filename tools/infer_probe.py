#!/usr/bin/env python3
"""Inferences/s of the batch inference (ModelContext.infer_batch: csrc/infer.cu on the int8 tensor cores) against the per-input device
path (dph_zkml_prove mode 1: run_device, the prover's witness inference), on seeded distinct inputs.
    usage: infer_probe.py [--models dense4m,cnn264k,cifar,covid] [--sizes 1024,8192] [--per-input 32] [--rounds 3] [--out FILE]
Each round runs every model's arms back to back (batch inference at each size, then the per-input path on --per-input inputs), after
one warm-up of each.  A last pass with the library's per-kernel timing on reads the GEMM kernel's time at the largest size and sets
the int8 operations it runs against the data sheet's 1,979 dense INT8 TOPS (H100 SXM, 700 W), and its bytes against 3.35 TB/s.
Prints one line per run and a JSON summary (median and range, the GPU's name, power limit and clocks) that --out also writes."""
import argparse, json, os, statistics, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
import dpb200 as dp
import models

ap = argparse.ArgumentParser()
ap.add_argument("--models", default="dense4m,cnn264k,cifar,covid")
ap.add_argument("--sizes", default="1024,8192")
ap.add_argument("--per-input", type=int, default=32)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--out")
a = ap.parse_args()
SIZES = [int(s) for s in a.sizes.split(",")]
INT8_TOPS, HBM_TBS = 1979.0, 3.35


def gpu_settings():
    import subprocess
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return dict(zip(q.split(","), [v.strip() for v in line.splitlines()[0].split(",")]))
    except Exception as e:
        return {"error": str(e)}


def dense4m():
    """bench.py's Dense-4M shape: 4 x [Dense 1024x1024 + bias -> Requant -> ReLU], weights and bias seeded in [-127, 127]"""
    nl, w = 4, 1024
    rng = np.random.Generator(np.random.PCG64(1))
    lw = w.bit_length() - 1
    fp = ((lw + 24 + 7) // 8) * 8 - lw
    rq = np.array([[lw, fp, 3 << (fp - 2), 2 * 7 + lw + 1]] * nl, dtype=np.int64)
    ctx = dp.ZkmlContext(nl, w, rng.integers(-127, 128, size=nl * w * w), rng.integers(-127, 128, size=nl * w), rq)
    return ctx, lambda n, s: np.random.Generator(np.random.PCG64(s)).integers(-127, 128, size=(n, w)).astype(np.int64)


def images(n_p, c_p, img):
    def draw(n, s):
        x = np.zeros((n, c_p, n_p, n_p), dtype=np.int64)
        x[:, :3, :img, :img] = np.random.Generator(np.random.PCG64(s)).integers(-127, 128, size=(n, 3, img, img))
        return x.reshape(n, -1)
    return draw


def build(name):
    if name == "dense4m":
        return dense4m()
    if name == "cnn264k":
        desc, data, x, _ = models.cnn(seed=1)
        return dp.ModelContext(desc, data, x.size), images(32, 4, 32)
    if name == "covid":
        desc, data, x, _ = models.covid(seed=1)
        return dp.ModelContext(desc, data, x.size), images(256, 4, 224)
    path = os.path.join(ROOT, "tests", "golden", "onnx", "cnn-cifar-01.onnx")
    ctx = dp.ModelContext.from_onnx(path, calibration=np.load(os.path.splitext(path)[0] + "-inputs.npz")["inputs"])
    md = ctx.metadata
    return ctx, lambda n, s: md.quantize_input(np.random.Generator(np.random.PCG64(s)).uniform(-1, 1, size=(n,) + md.input_shape).astype(np.float32))


dp.init(0)
summary = {"gpu": gpu_settings(), "sizes": SIZES, "per_input_inputs": a.per_input, "rounds": a.rounds, "models": {}}
print(summary["gpu"])
names = a.models.split(",")
ctxs = {n: build(n) for n in names}
xs = {n: draw(max(SIZES), 100) for n, (_, draw) in ctxs.items()}


def batch(name, size):
    sec, _, status, errors = ctxs[name][0].infer_batch(xs[name][:size])
    if (status != 0).any():
        raise SystemExit("%s: input failed: %s" % (name, next(e for e in errors if e)))
    return size / sec


def per_input(name):
    ctx = ctxs[name][0]
    t0 = time.perf_counter()
    for x in xs[name][: a.per_input]:
        ctx.run_inference(x)
    return a.per_input / (time.perf_counter() - t0)


for n in names:                       # warm-up: plans, modules, the per-input path's arena
    for s in SIZES:
        batch(n, s)
    per_input(n)
rates = {n: {**{"batch_%d" % s: [] for s in SIZES}, "per_input": []} for n in names}
for r in range(a.rounds):
    for n in names:
        for s in SIZES:
            rates[n]["batch_%d" % s].append(batch(n, s))
        rates[n]["per_input"].append(per_input(n))
        print("round %d %s: %s inferences/s" % (r, n, {k: round(v[-1], 1) for k, v in rates[n].items()}))
        sys.stdout.flush()

# the GEMM kernel's share of the tensor cores and of HBM at the largest size, from the library's per-kernel CUDA-event timing
s = max(SIZES)
for n in names:
    dp.profile_enable(True); dp.profile_reset()
    batch(n, s)
    dp.lib().dp_profile_flush()
    prof = dp.profile_read(with_units=True)
    dp.profile_enable(False)
    launches, ms, nbytes, ops = prof.get("k_infer_gemm", (0, 0.0, 0, 0))
    tops, tbs = ops / (ms * 1e-3) / 1e12, nbytes / (ms * 1e-3) / 1e12
    t_ops, t_bytes = ops / (INT8_TOPS * 1e12), nbytes / (HBM_TBS * 1e12)
    bound = "int8 tensor cores" if t_ops >= t_bytes else "HBM"
    floor_s = max(t_ops, t_bytes)
    rates[n]["gemm"] = {"batch": s, "launches": launches, "kernel_ms": ms, "int8_ops": ops, "bytes": nbytes, "tops": tops, "tb_per_s": tbs,
                        "bound": bound, "share_of_bound": floor_s / (ms * 1e-3) if ms else None}
    print("%s gemm at %d: %.2f ms over %d launches, %.1f TOPS (%.1f %% of %d), %.2f TB/s; %s-bound floor %.1f %%" % (
        n, s, ms, launches, tops, 100 * tops / INT8_TOPS, INT8_TOPS, tbs, bound, 100 * rates[n]["gemm"]["share_of_bound"]))

for n in names:
    summary["models"][n] = {k: ({"median": statistics.median(v), "min": min(v), "max": max(v)} if isinstance(v, list) else v) for k, v in rates[n].items()}
summary["gpu_after"] = gpu_settings()
for ctx, _ in ctxs.values():
    ctx.free()
print(json.dumps(summary))
if a.out:
    with open(a.out, "w") as f:
        json.dump(summary, f, indent=1)
