#!/usr/bin/env python3
"""Proofs/s of an imported ONNX model: ModelContext.from_onnx, then prove_batch on N distinct seeded float inputs in [-1, 1]
(quantised by the model's metadata), blocking wait mode.
    usage: onnx_probe.py [MODEL.onnx] [--workers 48] [--n 192] [--rounds 3] [--out FILE]
The default model is tests/golden/onnx/cnn-cifar-01.onnx.  Prints one line per run and a JSON summary (with the GPU's name,
power limit and clocks) that --out also writes."""
import argparse, json, os, statistics, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
import dpb200 as dp

ap = argparse.ArgumentParser()
ap.add_argument("model", nargs="?", default=os.path.join(ROOT, "tests", "golden", "onnx", "cnn-cifar-01.onnx"))
ap.add_argument("--workers", type=int, default=48)
ap.add_argument("--n", type=int, default=192)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--out")
a = ap.parse_args()


def gpu_settings():
    import subprocess
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return dict(zip(q.split(","), [v.strip() for v in line.splitlines()[0].split(",")]))
    except Exception as e:
        return {"error": str(e)}


dp.init(0)
dp.set_wait_mode(1)
ctx = dp.ModelContext.from_onnx(a.model)
xs = ctx.metadata.quantize_input(np.random.default_rng(2025).uniform(-1, 1, size=(a.n,) + ctx.metadata.input_shape).astype(np.float32))
summary = {"gpu": gpu_settings(), "model": os.path.basename(a.model), "wait_mode": "blocking", "workers": a.workers, "proofs_per_run": a.n}
print(summary["gpu"])
ctx.prove_batch(xs[: a.workers], a.workers)                    # warm the pool's threads and size the stride
rates = []
for r in range(a.rounds):
    sec, _, _, status, errors = ctx.prove_batch(xs, a.workers)
    if (status != 0).any():
        raise SystemExit("batch job failed: %s" % next(e for e in errors if e))
    rates.append(a.n / sec)
    print("round %d: %.1f proofs/s" % (r, rates[-1]))
    sys.stdout.flush()
summary["proofs_per_s"] = {"median": statistics.median(rates), "runs": rates}
summary["gpu_after"] = gpu_settings()
dp.host().dph_zkml_pool_free(ctx.h)
ctx.free()
print(json.dumps(summary))
if a.out:
    with open(a.out, "w") as f:
        json.dump(summary, f, indent=1)
