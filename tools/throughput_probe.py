#!/usr/bin/env python3
"""Where does multi-proof throughput saturate?  Dense-4M proofs/s and kernel launches/s against the number of proving threads
(each with its own stream + arena) on one GPU.
    usage: throughput_probe.py [dense4m|cnn264k] [workers ...] [--hasher poseidon2|blake3] [--wait spin|block]
--hasher blake3 proves under the `blake` feature (BlakeHasher + BlakeTranscript); --wait block lets the proving threads sleep on the
library's poller, the configuration in which the resident kernels run the transcript on the device."""
import argparse, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
import bench, dpb200 as dp
ap = argparse.ArgumentParser()
ap.add_argument("args", nargs="*")
ap.add_argument("--hasher", default="poseidon2", choices=["poseidon2", "blake3"])
ap.add_argument("--wait", default="spin", choices=["spin", "block"])
a = ap.parse_args()
which = a.args[0] if a.args and not a.args[0].isdigit() else "dense4m"
ws = [int(x) for x in a.args if x.isdigit()] or [1, 4, 8, 16, 24, 32, 48, 64]
wl = bench.DenseWorkload() if which == "dense4m" else bench.CnnWorkload()
dp.init(0); dp.set_hasher(1 if a.hasher == "blake3" else 0); wl.setup_device(dp); dp.set_wait_mode(1 if a.wait == "block" else 0)
print("%s, hasher %s, wait mode %s" % (which, a.hasher, a.wait))
def cpu_stat():
    d = {}
    try:
        for l in open("/sys/fs/cgroup/cpu.stat"):
            k, v = l.split(); d[k] = int(v)
    except Exception:
        pass
    return d
for nw in ws:
    n = max(16, 6 * nw)
    wl.ctx.prove_concurrent(nw, nw)            # warm the threads' pools
    l0 = dp.lib().dp_kernel_launches(); c0 = cpu_stat()
    sec = wl.ctx.prove_concurrent(nw, n)
    l1 = dp.lib().dp_kernel_launches(); c1 = cpu_stat()
    print("workers %2d: %3d proofs in %.3f s -> %6.1f proofs/s  (%.1f ms per proof per stream, %d launches/proof, %.0f k launches/s)"
          % (nw, n, sec, n / sec, 1e3 * sec * nw / n, (l1 - l0) // n, (l1 - l0) / sec / 1e3)
          + ("  | CPUs busy %.1f (user %.1f sys %.1f), %.1f CPU-ms per proof, throttled periods +%d" % (
              (c1["usage_usec"] - c0["usage_usec"]) / 1e6 / sec, (c1["user_usec"] - c0["user_usec"]) / 1e6 / sec, (c1["system_usec"] - c0["system_usec"]) / 1e6 / sec,
              (c1["usage_usec"] - c0["usage_usec"]) / 1e3 / n, c1["nr_throttled"] - c0["nr_throttled"]) if c0 and c1 else ""))
    sys.stdout.flush()
dp.host().dph_zkml_pool_free(wl.ctx.h)
