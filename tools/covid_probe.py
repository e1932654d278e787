#!/usr/bin/env python3
"""The covid vision model (models.covid(): 3x224x224, five 3x3 convolutions, 1,457,537 real parameters) on one GPU: single-proof
latency with spinning waits, proofs/s with blocking waits and as many proofs in flight as HBM holds, and the dp_profile time of the
long-row FFT (dp_fft_rows_long) with its achieved bytes/s against the H100 SXM's 3.35 TB/s.  The card's name and power limit are
read in the same run.  Prints one JSON line (and writes it to --json when given).
    usage: covid_probe.py [--channels 32,64,64,128,128] [--fc 64] [--proofs 3] [--max-inflight 16] [--check] [--json PATH]
--check also proves once on the CPU checker (tests/oracle_py.py) and compares the flat proofs; it reports the checker's time."""
import argparse, json, os, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import dpb200 as dp
import models

HBM_BPS = 3.35e12
ap = argparse.ArgumentParser()
ap.add_argument("--channels", default="32,64,64,128,128")
ap.add_argument("--fc", type=int, default=64)
ap.add_argument("--proofs", type=int, default=3, help="timed single proofs")
ap.add_argument("--max-inflight", type=int, default=16)
ap.add_argument("--check", action="store_true")
ap.add_argument("--json", default=None)
a = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
channels = tuple(int(c) for c in a.channels.split(","))
desc, data, x, n_params = models.covid(seed=1, channels=channels, fc=a.fc)
dp.init(0)
import torch
res = {"model": "covid", "channels": channels, "fc": a.fc, "real_params": n_params, "card": card}

t = time.perf_counter(); ctx = dp.ModelContext(desc, data, x.size); res["setup_s"] = time.perf_counter() - t
# latency, spinning waits (the default mode): end to end from the host input, inference included
dp.set_wait_mode(0)
first = ctx.prove(x)
lat = []
for _ in range(a.proofs):
    t = time.perf_counter(); ctx.prove(x); lat.append(time.perf_counter() - t)
res["latency_spin_ms"] = {"median": 1e3 * statistics.median(lat), "min": 1e3 * min(lat), "max": 1e3 * max(lat)}

# the long-row FFT in one proof
dp.profile_enable(True); dp.profile_reset()
ctx.prove(x)
prof = dp.profile_read(); dp.profile_enable(False); dp.profile_reset()
if "k_fft_long" in prof:
    n, ms, by = prof["k_fft_long"]
    res["k_fft_long"] = {"launches": n, "ms": ms, "bytes": by, "achieved_TBps": by / (ms * 1e-3) / 1e12, "of_3.35TBps": by / (ms * 1e-3) / HBM_BPS}
if "k_fft_rows" in prof:
    res["k_fft_rows_ms"] = prof["k_fft_rows"][1]

# throughput, blocking waits: one worker's footprint measured, then as many workers as 80% of the free HBM holds
dp.set_wait_mode(1)
ctx.run_inference(x)
free0 = torch.cuda.mem_get_info()[0]
ctx.prove_concurrent(1, 1)
free1 = torch.cuda.mem_get_info()[0]
per_worker = max(1, free0 - free1)
nw = max(1, min(a.max_inflight, 1 + int(0.8 * free1 // per_worker)))
ctx.prove_concurrent(nw, nw)                        # warm every worker's pool
n_proofs = 3 * nw
sec = ctx.prove_concurrent(nw, n_proofs)
res["throughput_block"] = {"in_flight": nw, "worker_bytes": per_worker, "proofs": n_proofs, "seconds": sec, "proofs_per_s": n_proofs / sec}
dp.set_wait_mode(0)

if a.check:
    import oracle_py as O
    t = time.perf_counter(); exp, _ = O.model_prove(desc, data, x, cap=1 << 25); res["checker_s"] = time.perf_counter() - t
    res["checker_equal"] = bool(exp.shape == first.shape and (exp == first).all())
ctx.free()
line = json.dumps(res)
print(line)
if a.json:
    os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
    open(a.json, "w").write(line + "\n")
