#!/usr/bin/env python3
"""Arrival-to-result latency and completed inputs/s: stacked streams (StackedContext.open_stream) at R = 8 and 64 against the plain
ProofStream on the base, on the same distinct inputs.  Arrivals are a seeded Poisson process at offered loads given as multiples of the
plain stream's capacity, measured in the same call (all inputs submitted at once).  Each arrival is submitted at its scheduled time and
a collector thread takes results; latency is from the scheduled time to the result in Python, inputs/s is arrivals over (last result -
first arrival).  Capacity: all inputs submitted at once to each stacked stream, against prove_stacked on the same inputs.  Screening:
the mean seconds of a group's infer_batch call, and their sum's share of the run.  Blocking waits; the arms alternate within each round.
    usage: stacked_stream_probe.py [dense4m] [iris] [--workers 48] [--r64-workers 8] [--n 480] [--loads 0.5,2,10] [--max-wait 0.02]
                                   [--rounds 3] [--out FILE]
Prints one line per run and a JSON summary (with the GPU's name, power limit and clocks, read before and after) that --out also
writes."""
import argparse, json, os, statistics, subprocess, sys, threading, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench, dpb200 as dp

ap = argparse.ArgumentParser()
ap.add_argument("workloads", nargs="*", default=["dense4m", "iris"])
ap.add_argument("--workers", type=int, default=48, help="workers of the plain stream and of the R = 8 stacked stream")
ap.add_argument("--r64-workers", type=int, default=8, help="workers of the R = 64 stacked stream (Dense-4M: 805 MB per thread)")
ap.add_argument("--n", type=int, default=480, help="arrivals per run")
ap.add_argument("--loads", default="0.5,2,10")
ap.add_argument("--max-wait", type=float, default=0.020)
ap.add_argument("--rounds", type=int, default=3)
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
    """(base context, [n, input_len] distinct seeded inputs), as stacked_probe.py draws them"""
    if key == "dense4m":
        wl = bench.DenseWorkload()
        ctx = dp.ZkmlContext(wl.NL, wl.W, wl.weights, wl.bias, wl.rq)
        return ctx, np.random.Generator(np.random.PCG64(2024)).integers(0, 128, size=(n, wl.W)).astype(np.int64)
    from test_onnx_calibration import GOLDEN, samples
    xs = samples("mlp-iris-01")[0]
    ctx = dp.ModelContext.from_onnx(os.path.join(GOLDEN, "mlp-iris-01.onnx"), calibration=xs)
    rng = np.random.Generator(np.random.PCG64(2024))
    f = np.clip(xs[rng.integers(0, len(xs), n)] + rng.uniform(-0.02, 0.02, size=(n,) + xs.shape[1:]), -1, 1).astype(np.float32)
    return ctx, ctx.metadata.quantize_input(f)


def sleep_until(t):
    d = t - time.perf_counter()
    if d > 0:
        time.sleep(d)


def run(open_stream, xs, arrivals):
    """-> (scheduled arrival times, result times, (groups screened, their seconds) or None); arrivals None: everything at once"""
    n = len(xs)
    done = np.zeros(n)
    submitted = threading.Semaphore(0)          # the collector calls next only with an input uncollected
    with open_stream() as s:
        def collect():
            for _ in range(n):
                submitted.acquire()
                r = s.next()
                if r.status:
                    raise SystemExit("stream input failed: %s" % r.error)
                done[r.ticket] = time.perf_counter()     # a fresh stream's tickets are the input indices
        th = threading.Thread(target=collect)
        t0 = time.perf_counter() + 0.05
        th.start()
        if arrivals is None:
            sleep_until(t0)
            s.submit(xs)
            for _ in range(n):
                submitted.release()
            arrived = np.full(n, t0)
        else:
            for i in range(n):
                sleep_until(t0 + arrivals[i])
                s.submit(xs[i])
                submitted.release()
            arrived = t0 + arrivals
        th.join()
        screen = (s.screen_calls, s.screen_seconds) if hasattr(s, "screen_calls") else None
    if not done.all():
        raise SystemExit("a stream lost results")
    return arrived, done, screen


def stats(arrived, done, screen):
    lat = 1e3 * (done - arrived)
    st = {"inputs_per_s": len(done) / (done.max() - arrived.min()),
          "p50_ms": float(np.percentile(lat, 50)), "p90_ms": float(np.percentile(lat, 90)), "p99_ms": float(np.percentile(lat, 99))}
    if screen:
        st.update(groups=screen[0], screen_ms_per_group=1e3 * screen[1] / screen[0], screen_share=screen[1] / (done.max() - arrived.min()))
    return st


def med_range(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}


dp.init(0)
dp.set_wait_mode(1)
summary = {"gpu": gpu_settings(), "wait_mode": "blocking", "workers": a.workers, "r64_workers": a.r64_workers, "arrivals_per_run": a.n,
           "loads_x_plain_capacity": LOADS, "max_wait_s": a.max_wait, "rounds": a.rounds, "workloads": {}}
print(summary["gpu"])
for key in a.workloads:
    ctx, xs = workload(key, a.n)
    assert (ctx.infer_batch(xs)[2] == 0).all()
    ctx.prove_batch(xs[: a.workers], a.workers)                   # warm the base pool's threads and size its stride
    sctx = {8: ctx.stacked(8), 64: ctx.stacked(64)}
    workers = {"plain": a.workers, "R8": a.workers, "R64": a.r64_workers}
    for R, sc in sctx.items():                                     # warm each stacked pool's threads and size its stride
        w = workers["R%d" % R]
        sc.prove_stacked(np.concatenate([xs] * (-(-R * w // a.n)))[: R * w], w)
    opens = {"plain": lambda: ctx.open_stream(a.workers, capacity=a.n),
             "R8": lambda: sctx[8].open_stream(a.workers, a.max_wait, capacity=a.n),
             "R64": lambda: sctx[64].open_stream(a.r64_workers, a.max_wait, capacity=a.n)}
    cap = {arm: [] for arm in opens}
    cap_stacked = {"R8": [], "R64": []}
    for r in range(2):                                             # capacity: all inputs at once
        for arm in opens:
            cap[arm].append(stats(*run(opens[arm], xs, None))["inputs_per_s"])
        for arm, R in (("R8", 8), ("R64", 64)):
            t = time.perf_counter()
            out = sctx[R].prove_stacked(xs, workers[arm])
            assert (out[4] == 0).all()
            cap_stacked[arm].append(a.n / (time.perf_counter() - t))
    rate = statistics.median(cap["plain"])
    print("%s capacity, inputs/s: %s; prove_stacked %s" % (key, {k: ["%.0f" % v for v in c] for k, c in cap.items()},
                                                          {k: ["%.0f" % v for v in c] for k, c in cap_stacked.items()}))
    res = {load: {arm: [] for arm in opens} for load in LOADS}
    for r in range(a.rounds):
        for li, load in enumerate(LOADS):
            arrivals = np.cumsum(np.random.default_rng(1000 * r + li).exponential(1.0 / (load * rate), size=a.n))
            arms = list(opens)[(r + li) % 3:] + list(opens)[: (r + li) % 3]
            for arm in arms:
                st = stats(*run(opens[arm], xs, arrivals))
                res[load][arm].append(st)
                print("%s round %d load %.1fx %-5s: %.0f inputs/s, latency p50 %.0f ms, p90 %.0f ms, p99 %.0f ms%s"
                      % (key, r, load, arm, st["inputs_per_s"], st["p50_ms"], st["p90_ms"], st["p99_ms"],
                         "" if "groups" not in st else ", %d groups, screening %.2f ms per group (%.1f %% of the run)"
                         % (st["groups"], st["screen_ms_per_group"], 100 * st["screen_share"])))
                sys.stdout.flush()
    summary["workloads"][key] = {
        "plain_capacity_inputs_per_s": med_range(cap["plain"]),
        "stream_capacity_inputs_per_s": {arm: med_range(v) for arm, v in cap.items()},
        "prove_stacked_inputs_per_s": {arm: med_range(v) for arm, v in cap_stacked.items()},
        "loads": {str(load): {arm: {k: med_range([s[k] for s in runs]) for k in runs[0]} for arm, runs in v.items()} for load, v in res.items()}}
    for sc in sctx.values():
        sc.free()
    ctx.free()
summary["gpu_after"] = gpu_settings()
print(json.dumps(summary))
if a.out:
    with open(a.out, "w") as f:
        json.dump(summary, f, indent=1)
