#!/usr/bin/env python3
"""Distinct inputs against the repeated stored input: proofs/s of dph_zkml_prove_batch (N different seeded inputs, each proved end
to end and returning its output) and of prove_concurrent(e2e=True) (N proofs of the one stored input), alternating the two arms in
one process, blocking wait mode, the same worker count.
    usage: batch_probe.py [dense4m] [cnn264k] [--workers 48] [--n 192] [--rounds 3] [--out FILE]
Prints one line per run and a JSON summary (with the GPU's name, power limit and clocks) that --out also writes."""
import argparse, json, os, statistics, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
import bench, dpb200 as dp, models

ap = argparse.ArgumentParser()
ap.add_argument("workloads", nargs="*", default=["dense4m", "cnn264k"])
ap.add_argument("--workers", type=int, default=48)
ap.add_argument("--n", type=int, default=192)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--out")
a = ap.parse_args()


def gpu_settings():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return dict(zip(q.split(","), [v.strip() for v in line.splitlines()[0].split(",")]))
    except Exception as e:
        return {"error": str(e)}


def inputs(key, wl, n):
    """n distinct seeded inputs in the workload's input layout"""
    if key == "dense4m":
        rng = np.random.Generator(np.random.PCG64(2024))
        return rng.integers(0, 128, size=(n, wl.x.size)).astype(np.int64)     # the range of the stored input's draw (% 128)
    return np.stack([models.cnn(seed=1000 + j)[2] for j in range(n)]).astype(np.int64)   # CNN-264k's padded layout, other seeds


dp.init(0)
dp.set_wait_mode(1)
summary = {"gpu": gpu_settings(), "wait_mode": "blocking", "workers": a.workers, "proofs_per_run": a.n, "workloads": {}}
print(summary["gpu"])
for key in a.workloads:
    wl = bench.DenseWorkload() if key == "dense4m" else bench.CnnWorkload()
    wl.setup_device(dp)
    xs = inputs(key, wl, a.n)
    ctx = wl.ctx
    ctx.prove_batch(xs[: a.workers], a.workers)                 # warm the pool's threads and size the stride
    ctx.prove_concurrent(a.workers, a.workers, e2e=True)
    rates = {"batch": [], "e2e": []}
    for r in range(a.rounds):
        sec, proofs, _, status, errors = ctx.prove_batch(xs, a.workers)
        if (status != 0).any():
            raise SystemExit("%s: batch job failed: %s" % (key, next(e for e in errors if e)))
        rates["batch"].append(a.n / sec)
        sec_e2e = ctx.prove_concurrent(a.workers, a.n, e2e=True)
        rates["e2e"].append(a.n / sec_e2e)
        print("%s round %d: distinct inputs %.1f proofs/s, stored input e2e %.1f proofs/s" % (key, r, rates["batch"][-1], rates["e2e"][-1]))
        sys.stdout.flush()
    summary["workloads"][key] = {k: {"median": statistics.median(v), "runs": v} for k, v in rates.items()}
    dp.host().dph_zkml_pool_free(ctx.h)
    ctx.free()
summary["gpu_after"] = gpu_settings()
print(json.dumps(summary))
if a.out:
    with open(a.out, "w") as f:
        json.dump(summary, f, indent=1)
