#!/usr/bin/env python3
"""CUDA runtime API census of W concurrent Dense-4M proofs: calls per proof and time the proving threads spend inside each call
(CUPTI callbacks; kernel-timeline tracing stays off).  usage: trace_api.py [workers] [proofs] [wait mode: 0 spin (default) | 1 block]
-> api_w<workers>_mode<mode>.csv in the current directory + a summary"""
import ctypes as C, os, sys, csv
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
import bench, dpb200 as dp
W = int(sys.argv[1]) if len(sys.argv) > 1 else 16
N = int(sys.argv[2]) if len(sys.argv) > 2 else 2 * W
MODE = int(sys.argv[3]) if len(sys.argv) > 3 else 0
T = C.CDLL(os.path.join(ROOT, "deep-prove_b200", "libdp_trace.so"))
T.dp_trace_api_stop.argtypes = [C.c_char_p]
dp.set_wait_mode(MODE)
wl = bench.DenseWorkload(); dp.init(0); wl.setup_device(dp)
wl.ctx.prove_concurrent(W, W)
assert T.dp_trace_api_start() == 0
sec = wl.ctx.prove_concurrent(W, N)
path = os.path.abspath("api_w%d_mode%d.csv" % (W, MODE))
T.dp_trace_api_stop(path.encode())
rows = sorted(csv.DictReader(open(path)), key=lambda r: -float(r["total_ms"]))
tot = sum(float(r["total_ms"]) for r in rows)
print("workers %d: %d proofs in %.3f s -> %.1f proofs/s (API callbacks on); thread-time inside CUDA runtime calls: %.1f ms per proof (%.1f CPUs)" % (W, N, sec, N / sec, tot / N, tot / 1e3 / sec))
for r in rows[:14]:
    print("  %-34s %8.1f calls/proof  %9.2f ms/proof  mean %7.2f us" % (r["api"], float(r["calls"]) / N, float(r["total_ms"]) / N, float(r["mean_us"])))
