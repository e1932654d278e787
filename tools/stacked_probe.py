#!/usr/bin/env python3
"""Stacked proofs against one proof per input: inputs proved per second end to end by StackedContext.prove_stacked (screening,
grouping, R inputs per proof) and by prove_batch on the same distinct inputs, alternating the arms in one process, blocking wait mode.
Per stacked proof it also reports the latency (one group alone on one worker), the proof words per input, the per-kernel times of
one proof (the library's CUDA-event profile, k_wit_matmul's share among them), and the device memory one
proving thread holds after a proof (its arena keeps the slabs it grew to, so this covers the proof's peak); the stacked arm's worker
counts are capped by what the free device memory holds at that size, and the cap is reported.
    usage: stacked_probe.py [dense4m] [iris] [--R 1,8,64,256] [--workers 48] [--stacked-workers 8,48] [--n 512] [--rounds 3] [--out FILE]
Each stacked arm proves max(n, R * workers) inputs.  Prints one line per run and a JSON summary (with the GPU's name, power limit and
clocks before and after) that --out also writes."""
import argparse, json, os, statistics, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench, dpb200 as dp, models

ap = argparse.ArgumentParser()
ap.add_argument("workloads", nargs="*", default=["dense4m", "iris"])
ap.add_argument("--R", default="1,8,64,256")
ap.add_argument("--workers", type=int, default=48)
ap.add_argument("--stacked-workers", default="8,48")
ap.add_argument("--n", type=int, default=512)
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


def used_bytes():
    import torch
    free, total = torch.cuda.mem_get_info(0)
    return total - free, free


def workload(key, n):
    """(base context, [n, input_len] distinct seeded inputs)"""
    if key == "dense4m":
        wl = bench.DenseWorkload()
        ctx = dp.ZkmlContext(wl.NL, wl.W, wl.weights, wl.bias, wl.rq)
        return ctx, np.random.Generator(np.random.PCG64(2024)).integers(0, 128, size=(n, wl.W)).astype(np.int64)
    from test_onnx_calibration import GOLDEN, samples
    xs = samples("mlp-iris-01")[0]
    ctx = dp.ModelContext.from_onnx(os.path.join(GOLDEN, "mlp-iris-01.onnx"), calibration=xs)
    rng = np.random.Generator(np.random.PCG64(2024))        # the reference's 30 samples, each drawn many times with a little noise
    f = np.clip(xs[rng.integers(0, len(xs), n)] + rng.uniform(-0.02, 0.02, size=(n,) + xs.shape[1:]), -1, 1).astype(np.float32)
    return ctx, ctx.metadata.quantize_input(f)


def timed(call):
    t = time.perf_counter()
    r = call()
    return time.perf_counter() - t, r


dp.init(0)
dp.set_wait_mode(1)
Rs = [int(v) for v in a.R.split(",")]
s_workers = sorted(int(v) for v in a.stacked_workers.split(","))
summary = {"gpu": gpu_settings(), "wait_mode": "blocking", "batch_workers": a.workers, "rounds": a.rounds, "workloads": {}}
print(summary["gpu"])
for key in a.workloads:
    n_max = max([a.n] + [R * w for R in Rs for w in s_workers])
    ctx, xs_all = workload(key, n_max)
    xs = xs_all[: a.n]
    st = ctx.infer_batch(xs_all)[2]
    ok = int((st[: a.n] == 0).sum())
    ctx.prove_batch(xs[: a.workers], a.workers)          # warm the pool's threads and size the stride
    res = {"inputs": a.n, "screened_out": a.n - ok, "batch": {"runs": []}, "stacked": {}}
    for R in Rs:
        u0, _ = used_bytes()
        try:
            t_setup, sctx = timed(lambda: ctx.stacked(R))
        except dp.DpError as e:                               # a size the device memory does not hold: recorded as the limit
            res["stacked"][str(R)] = {"R": R, "error": str(e)}
            print("%s R=%d: %s" % (key, R, e))
            continue
        u1, free = used_bytes()
        lat, out = timed(lambda: sctx.prove_stacked(xs_all[:R], 1, stride=1 << 25))
        if (out[4] != 0).any():                               # a proof the device memory does not hold fails its job
            res["stacked"][str(R)] = {"R": R, "error": next(e for e in out[5] if e)}
            print("%s R=%d: %s" % (key, R, res["stacked"][str(R)]["error"]))
            dp.host().dph_zkml_pool_free(sctx.h)
            sctx.free()
            continue
        lat, out = timed(lambda: sctx.prove_stacked(xs_all[:R], 1, stride=1 << 25))   # the thread's arena is grown: latency alone
        u2, free = used_bytes()
        words = int(out[1][0].size)
        dp.profile_enable(True); dp.profile_reset()              # per-kernel CUDA-event times of one proof on this thread
        sctx.prove(models.pad_rows(xs_all[:R], R))
        prof = dp.profile_read(cap=128); dp.profile_enable(False); dp.profile_reset()
        top = sorted(prof.items(), key=lambda kv: -kv[1][1])[:6]
        per_thread = max(u2 - u1, 1)
        w_cap = max(1, int(0.85 * free / per_thread) + 1)   # the thread already running holds its share
        arm = {"R": R, "setup_s": t_setup, "setup_bytes": u1 - u0, "latency_s": lat, "proof_words": words, "words_per_input": words / R,
               "bytes_per_thread": per_thread, "worker_cap": w_cap, "profiled_ms": sum(v[1] for v in prof.values()),
               "k_wit_matmul_ms": prof.get("k_wit_matmul", (0, 0.0))[1], "top_kernels_ms": {k: v[1] for k, v in top}, "by_workers": {}}
        print("%s R=%d: setup %.2f s (%.0f MB), one proof %.1f ms alone, %d words (%.0f per input), %.0f MB per proving thread, "
              "memory holds %d threads" % (key, R, t_setup, (u1 - u0) / 1e6, lat * 1e3, words, words / R, per_thread / 1e6, w_cap))
        print("%s R=%d: profiled kernels %.1f ms, k_wit_matmul %.2f ms; top %s" % (key, R, arm["profiled_ms"], arm["k_wit_matmul_ms"],
              ", ".join("%s %.1f" % kv for kv in arm["top_kernels_ms"].items())))
        sys.stdout.flush()
        for w in s_workers:
            w_used = min(w, w_cap)
            n_s = max(a.n, R * w_used)
            xs_s = xs_all[:n_s]
            ok_s = int((st[:n_s] == 0).sum())
            sctx.prove_stacked(xs_s[: R * w_used], w_used, stride=words + 4096)       # grow this many threads' arenas
            runs = []
            for r in range(a.rounds):
                if w == s_workers[0]:                         # prove_batch alternates with each R's first stacked arm
                    sec, (_, _, _, status, _) = timed(lambda: ctx.prove_batch(xs, a.workers))
                    res["batch"]["runs"].append(int((status == 0).sum()) / sec)
                    print("%s prove_batch round %d: %.1f inputs/s" % (key, r, res["batch"]["runs"][-1]))
                sec, out = timed(lambda: sctx.prove_stacked(xs_s, w_used, stride=words + 4096))
                if (out[4][st[:n_s] == 0] != 0).any():
                    raise SystemExit("%s R=%d: a stacked proof failed: %s" % (key, R, next(e for e in out[5] if e)))
                runs.append(ok_s / sec)
                print("%s R=%d workers=%d round %d: %.1f inputs/s (%d inputs, %d proofs)" % (key, R, w_used, r, runs[-1], n_s, len(out[1])))
                sys.stdout.flush()
            arm["by_workers"][str(w_used)] = {"inputs": n_s, "median": statistics.median(runs), "runs": runs}
        res["stacked"][str(R)] = arm
        dp.host().dph_zkml_pool_free(sctx.h)
        sctx.free()
    res["batch"]["median"] = statistics.median(res["batch"]["runs"])
    summary["workloads"][key] = res
    dp.host().dph_zkml_pool_free(ctx.h)
    ctx.free()
summary["gpu_after"] = gpu_settings()
print(json.dumps(summary))
if a.out:
    with open(a.out, "w") as f:
        json.dump(summary, f, indent=1)
