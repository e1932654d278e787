"""Kernel launches and host waits per proof with many proofs in flight (the bench's configuration: blocking waits, STREAMS proofs per
GPU), from the library's process-wide counters dp_kernel_launches and dp_host_waits, plus the per-kernel launch counts of the profile.

    python tools/count_waits.py [--workload dense4m|cnn264k] [--hasher poseidon2|blake3] [--steps 2] [--json OUT]

--hasher blake3 proves under the `blake` feature (BlakeHasher Merkle trees, BlakeTranscript).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))

import bench  # noqa: E402
import dpb200 as dp  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="dense4m", choices=list(bench.WORKLOADS))
    ap.add_argument("--hasher", default="poseidon2", choices=["poseidon2", "blake3"])
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dp.init(0)
    dp.set_hasher(1 if a.hasher == "blake3" else 0)
    w = bench.WORKLOADS[a.workload]()
    w.setup_device(dp)
    dp.set_wait_mode(1)
    w.run_resident(1, 0)                                   # warm-up batch
    proofs = a.steps * w.units_per_step
    dp.profile_enable(True)
    dp.profile_reset()
    l0, h0 = dp.lib().dp_kernel_launches(), dp.lib().dp_host_waits()
    w.run_resident(a.steps, 0)
    launches, waits = dp.lib().dp_kernel_launches() - l0, dp.lib().dp_host_waits() - h0
    dp.lib().dp_profile_flush()
    prof = dp.profile_read(cap=128)
    dp.profile_enable(False)
    out = {"workload": a.workload, "hasher": a.hasher, "proofs": proofs, "launches_per_proof": launches / proofs, "host_waits_per_proof": waits / proofs,
           "kernel_launches_per_proof": {k: v[0] / proofs for k, v in sorted(prof.items())}}
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
