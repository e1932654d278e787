#!/usr/bin/env python3
"""Arrival-to-proof latency under load: one proof stream against a batching loop over prove_batch, on the same distinct inputs.
Arrivals are a seeded Poisson process at offered loads given as fractions of the prove_batch rate measured in the same call.
    (a) stream:   each arrival is submitted to one open ProofStream at once; a collector thread takes results as they finish.
    (b) batching: arrivals are collected until --batch of them are waiting or --window seconds passed since the first, then proved
                  by one prove_batch call (the batch's proofs all complete when the call returns).
For each arm: completed proofs/s (arrivals / (last completion - first arrival)) and the latency from an arrival's scheduled time
to its proof at p50, p90 and p99.  Blocking wait mode, the same worker pool for both arms, the arms alternating within each round.
    usage: stream_probe.py [dense4m] [cifar] [--workers 48] [--n 240] [--loads 0.5,0.8,0.95] [--rounds 3] [--out FILE]
Prints one line per run and a JSON summary (with the GPU's name, power limit and clocks, read before and after) that --out also
writes."""
import argparse, json, os, statistics, subprocess, sys, threading, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
import bench, dpb200 as dp

ap = argparse.ArgumentParser()
ap.add_argument("workloads", nargs="*", default=["dense4m", "cifar"])
ap.add_argument("--workers", type=int, default=48)
ap.add_argument("--n", type=int, default=240, help="arrivals per run")
ap.add_argument("--loads", default="0.5,0.8,0.95")
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--batch", type=int, default=48)
ap.add_argument("--window", type=float, default=0.020)
ap.add_argument("--out")
a = ap.parse_args()
LOADS = [float(v) for v in a.loads.split(",")]


def gpu_settings():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return dict(zip(q.split(","), [v.strip() for v in line.splitlines()[0].split(",")]))
    except Exception as e:
        return {"error": str(e)}


def workload(key, n):
    """(context, n distinct seeded inputs in its input layout)"""
    if key == "dense4m":
        wl = bench.DenseWorkload()
        wl.setup_device(dp)
        rng = np.random.Generator(np.random.PCG64(2024))
        return wl.ctx, rng.integers(0, 128, size=(n, wl.x.size)).astype(np.int64)
    path = os.path.join(ROOT, "tests", "golden", "onnx", "cnn-cifar-01.onnx")
    ctx = dp.ModelContext.from_onnx(path, calibration=np.load(os.path.splitext(path)[0] + "-inputs.npz")["inputs"])
    x = np.random.default_rng(2025).uniform(-1, 1, size=(n,) + ctx.metadata.input_shape).astype(np.float32)
    return ctx, ctx.metadata.quantize_input(x)


def sleep_until(t):
    d = t - time.perf_counter()
    if d > 0:
        time.sleep(d)


def run_stream(ctx, xs, arrivals):
    """-> (scheduled arrival times, completion times) indexed by input"""
    n = len(xs)
    done = np.zeros(n)
    submitted = threading.Semaphore(0)     # one release per submit: the collector calls next only with a job uncollected, since
    with ctx.open_stream(a.workers, capacity=n) as s:     # next on a stream with nothing in flight is refused at once
        def collect():
            for _ in range(n):
                submitted.acquire()
                r = s.next()
                if r.status:
                    raise SystemExit("stream job failed: %s" % r.error)
                done[r.ticket] = time.perf_counter()      # a fresh stream's tickets are the input indices
        t0 = time.perf_counter() + 0.05
        th = threading.Thread(target=collect)
        th.start()
        for i in range(n):
            sleep_until(t0 + arrivals[i])
            s.submit(xs[i])
            submitted.release()
        th.join()
    if not done.all():
        raise SystemExit("the stream arm lost results")
    return t0 + arrivals, done


def run_batching(ctx, xs, arrivals):
    n = len(xs)
    done = np.zeros(n)
    cv, pending = threading.Condition(), []
    t0 = time.perf_counter() + 0.05

    def batcher():
        k = 0
        while k < n:
            with cv:
                cv.wait_for(lambda: pending)
                deadline = t0 + arrivals[pending[0]] + a.window     # the oldest waiting arrival waits at most the window for company
                while len(pending) < a.batch and time.perf_counter() < deadline and pending[-1] < n - 1:
                    cv.wait(max(0.0, deadline - time.perf_counter()))
                take, pending[:] = pending[: a.batch], pending[a.batch:]
            _, _, _, status, errors = ctx.prove_batch(xs[take], a.workers)
            if (status != 0).any():
                raise SystemExit("batch job failed: %s" % next(e for e in errors if e))
            done[take] = time.perf_counter()
            k += len(take)
    th = threading.Thread(target=batcher)
    th.start()
    for i in range(n):
        sleep_until(t0 + arrivals[i])
        with cv:
            pending.append(i)
            cv.notify()
    th.join()
    return t0 + arrivals, done


def stats(arrived, done):
    lat = 1e3 * (done - arrived)
    return {"proofs_per_s": len(done) / (done.max() - arrived.min()),
            "p50_ms": float(np.percentile(lat, 50)), "p90_ms": float(np.percentile(lat, 90)), "p99_ms": float(np.percentile(lat, 99))}


def med_range(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}


dp.init(0)
dp.set_wait_mode(1)
summary = {"gpu": gpu_settings(), "wait_mode": "blocking", "workers": a.workers, "arrivals_per_run": a.n, "loads": LOADS,
           "batching": {"batch": a.batch, "window_s": a.window}, "workloads": {}}
print(summary["gpu"])
for key in a.workloads:
    ctx, xs = workload(key, a.n)
    ctx.prove_batch(xs[: a.workers], a.workers)                  # warm the pool's threads and size the stride
    rates = []
    for _ in range(2):
        sec, _, _, status, _ = ctx.prove_batch(xs, a.workers)
        assert (status == 0).all()
        rates.append(a.n / sec)
    rate = statistics.median(rates)
    print("%s: prove_batch of %d inputs: %s proofs/s" % (key, a.n, ["%.1f" % r for r in rates]))
    res = {load: {"stream": [], "batching": []} for load in LOADS}
    for r in range(a.rounds):
        for li, load in enumerate(LOADS):
            arrivals = np.cumsum(np.random.default_rng(1000 * r + li).exponential(1.0 / (load * rate), size=a.n))
            arms = ["stream", "batching"] if (r + li) % 2 == 0 else ["batching", "stream"]
            for arm in arms:
                st = stats(*(run_stream if arm == "stream" else run_batching)(ctx, xs, arrivals))
                res[load][arm].append(st)
                print("%s round %d load %.2f %-8s: %.1f proofs/s, latency p50 %.0f ms, p90 %.0f ms, p99 %.0f ms"
                      % (key, r, load, arm, st["proofs_per_s"], st["p50_ms"], st["p90_ms"], st["p99_ms"]))
                sys.stdout.flush()
    summary["workloads"][key] = {
        "prove_batch_proofs_per_s": med_range(rates),
        "loads": {str(load): {arm: {k: med_range([s[k] for s in runs]) for k in runs[0]} for arm, runs in v.items()} for load, v in res.items()}}
    ctx.free()
summary["gpu_after"] = gpu_settings()
print(json.dumps(summary))
if a.out:
    with open(a.out, "w") as f:
        json.dump(summary, f, indent=1)
