#!/usr/bin/env python3
"""Proofs/s of an imported ONNX model: ModelContext.from_onnx, then prove_batch on N distinct seeded float inputs in [-1, 1]
(quantised by the model's metadata), blocking wait mode.
    usage: onnx_probe.py [MODEL.onnx] [--quantization absmax|calibrated|both] [--workers 48] [--n 192] [--rounds 3] [--out FILE]
The default model is tests/golden/onnx/cnn-cifar-01.onnx.  --quantization calibrated imports it calibrated on the samples of
<model>-inputs.npz beside it (InferenceObserver); both runs the AbsoluteMax and the calibrated model, alternating them round by
round.  Prints one line per run and a JSON summary (with the GPU's name, power limit and clocks) that --out also writes."""
import argparse, json, os, statistics, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
import dpb200 as dp

ap = argparse.ArgumentParser()
ap.add_argument("model", nargs="?", default=os.path.join(ROOT, "tests", "golden", "onnx", "cnn-cifar-01.onnx"))
ap.add_argument("--quantization", choices=["absmax", "calibrated", "both"], default="absmax")
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
arms = ["absmax", "calibrated"] if a.quantization == "both" else [a.quantization]
ctxs, xs = {}, {}
for arm in arms:
    cal = np.load(os.path.splitext(a.model)[0] + "-inputs.npz")["inputs"] if arm == "calibrated" else None
    ctxs[arm] = ctx = dp.ModelContext.from_onnx(a.model, calibration=cal)
    xs[arm] = ctx.metadata.quantize_input(np.random.default_rng(2025).uniform(-1, 1, size=(a.n,) + ctx.metadata.input_shape).astype(np.float32))
summary = {"gpu": gpu_settings(), "model": os.path.basename(a.model), "wait_mode": "blocking", "workers": a.workers, "proofs_per_run": a.n}
print(summary["gpu"])
for arm in arms:
    ctxs[arm].prove_batch(xs[arm][: a.workers], a.workers)        # warm the pool's threads and size the stride
rates = {arm: [] for arm in arms}
words = {}
for r in range(a.rounds):
    for arm in arms:
        sec, proofs, _, status, errors = ctxs[arm].prove_batch(xs[arm], a.workers)
        if (status != 0).any():
            raise SystemExit("batch job failed: %s" % next(e for e in errors if e))
        rates[arm].append(a.n / sec)
        words[arm] = statistics.median(len(p) for p in proofs)
        print("round %d %s: %.1f proofs/s" % (r, arm, rates[arm][-1]))
        sys.stdout.flush()
summary["proofs_per_s"] = {arm: {"median": statistics.median(v), "runs": v, "proof_words_median": words[arm]} for arm, v in rates.items()}
summary["gpu_after"] = gpu_settings()
for ctx in ctxs.values():
    dp.host().dph_zkml_pool_free(ctx.h)
    ctx.free()
print(json.dumps(summary))
if a.out:
    with open(a.out, "w") as f:
        json.dump(summary, f, indent=1)
