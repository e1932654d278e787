#!/usr/bin/env python3
"""Per-round latency of the device sumcheck (host wall clock around dp_sc_round, which returns when the round message has arrived):
fixed challenges, no Fiat-Shamir in the loop.  usage: sc_rounds.py [nv] [resident 0|1] [shape: b3|e3|b2|logup]"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200")); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import dpb200 as dp
import bench
nv = int(sys.argv[1]) if len(sys.argv) > 1 else 20
resident = int(sys.argv[2]) if len(sys.argv) > 2 else 1
shape = sys.argv[3] if len(sys.argv) > 3 else "b3"
dp.init(0)
n = 1 << nv
def base(seed): return bench.splitmix_f(seed, n)
def ext(seed): return bench.splitmix_f(seed, 2 * n).reshape(n, 2)
if shape == "b3": mles = [(base(1), False), (base(2), False), (base(3), False)]; products = [((1, 0), [0, 1, 2])]
elif shape == "b2": mles = [(base(1), False), (base(2), False)]; products = [((1, 0), [0, 1])]
elif shape == "e3": mles = [(ext(1), True), (ext(2), True), (ext(3), True)]; products = [((1, 0), [0, 1, 2])]
else:   # logup-like: eq shared by three products over two instances
    mles = [(ext(1), True)] + [(ext(2 + i), True) for i in range(8)]
    products = [((1, 0), [0, 1, 2]), ((3, 1), [0, 3, 4]), ((5, 0), [0, 2, 4]), ((1, 0), [0, 5, 6]), ((3, 1), [0, 7, 8]), ((5, 0), [0, 6, 8])]
ch = bench.splitmix_f(99, 2 * nv).reshape(nv, 2)
deg = max(len(p[1]) for p in products)
for rep in range(3):
    dm = [dp.Mle.upload(a, e) for a, e in mles]
    sc = dp.Sumcheck(dm, products, nv, deg)
    dp.check(dp.lib().dp_sc_set_resident_tail(sc.h, resident))
    dp.lib().dp_synchronize()
    ts = []
    import ctypes as C
    out = np.zeros(2 * (deg + 1), dtype=np.uint64); po = out.ctypes.data_as(C.c_void_p)
    chp = [np.ascontiguousarray(ch[r]).ctypes.data_as(C.c_void_p) for r in range(nv)]
    f = dp.lib().dp_sc_round
    pc = time.perf_counter
    for r in range(nv):
        t0 = pc()
        rc = f(sc.h, None if r == 0 else chp[r - 1], po)
        ts.append((pc() - t0) * 1e6)
        assert rc == 0, dp.lib().dp_last_error()
    sc.finish(ch[nv - 1]); sc.destroy()
    if rep == 2:
        print("nv=%d shape=%s resident=%d total %.1f us; per round (us): %s" % (nv, shape, resident, sum(ts), " ".join("%.1f" % t for t in ts)))
