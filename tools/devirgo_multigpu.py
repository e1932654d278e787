#!/usr/bin/env python3
"""Single-proof sumcheck sharded over N GPUs (SURVEY 8(e) "single-sumcheck sharding", cfg 5B) -- run under torchrun:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29701 tools/devirgo_multigpu.py [nv] [reps]
Every rank owns a contiguous 1/N of each MLE on its own GPU; per round: one local launch + one NCCL all-gather of the
partial message.  Prints one JSON line: latency of the sharded proof (device events, max over ranks), the latency of the
same proof on one GPU (rank 0, when it fits), and whether the two proofs are bit-identical."""
import json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
import torch, torch.distributed as dist
import dpb200 as dp
import multigpu as mg


def splitmix_f(seed, n, skip=0):
    """n draws of splitmix64(seed) mod p starting at draw `skip` (vectorised; same stream as the bench inputs)"""
    i = np.arange(skip + 1, skip + n + 1, dtype=np.uint64)
    z = np.uint64(seed) + i * np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    return np.where(z >= np.uint64(mg.P), z - np.uint64(mg.P), z)


def main():
    nv = int(sys.argv[1]) if len(sys.argv) > 1 else 26
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    rank, world, local_rank = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local_rank)
    backend = os.environ.get("DP_DIST_BACKEND", "nccl")
    dist.init_process_group(backend, device_id=torch.device("cuda", local_rank) if backend == "nccl" else None)
    dp.init(local_rank); dp.use_torch_stream()
    ag = mg.TorchAllGather(dist)
    exch = os.environ.get("DP_EXCHANGE", "shm")     # shm: same-node mailbox (default); nccl: all-gather over NVLink; py: Python round loop + all-gather
    mb = mg.ShmMailbox("dpb200_devirgo_%d" % os.getppid(), rank, world, dist.barrier) if exch == "shm" else None
    n = 1 << nv
    lo, hi = mg.shard_range(n, rank, world)
    products = [((1, 0), [0, 1, 2])]
    slices = [splitmix_f(s, hi - lo, skip=lo) for s in (1, 2, 3)]

    def sharded():
        mles = [dp.Mle.upload(a, False) for a in slices]
        torch.cuda.synchronize(); dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if exch == "py": out = mg.prove_sharded_device(mles, products, nv, rank, world, ag)
        else: out = mg.prove_sharded_native(mles, products, nv, rank, world, mailbox=mb, allgather=None if mb is not None else ag)
        e1.record(); torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device="cuda" if backend == "nccl" else "cpu")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return out, float(t.item())

    sharded()                                                   # warm-up (NCCL channels, pools)
    runs = [sharded() for _ in range(reps)]
    ms = min(r[1] for r in runs)
    point, msgs, fin = runs[-1][0]
    single_ms, same = None, None
    if rank == 0 and 3 * 8 * n <= 32 << 30:      # the inputs plus the first folded tables (as large again) within 80 GB
        full = [splitmix_f(s, n) for s in (1, 2, 3)]
        ts = []
        for _ in range(max(3, reps // 2) + 1):             # first run grows the device arena (cudaMalloc): take the best
            mles = [dp.Mle.upload(a, False) for a in full]
            torch.cuda.synchronize(); t0 = time.perf_counter()
            ref = dp.sumcheck_prove_parallel(mles, products, nv)
            torch.cuda.synchronize(); ts.append(1e3 * (time.perf_counter() - t0))
        single_ms = min(ts)
        same = bool((ref[0] == point).all() and (ref[1] == msgs).all() and (ref[2] == fin).all())
    dist.barrier()
    if rank == 0:
        print(json.dumps({"workload": "sumcheck nv=%d deg=3 3xBase, ONE proof sharded over %d GPUs (devirgo split), backend %s" % (nv, world, backend),
                          "n_gpus": world, "exchange": exch, "sharded_ms": ms, "single_gpu_ms": single_ms, "bit_identical_to_single_gpu_proof": same,
                          "rounds": int(msgs.shape[0]), "exchange_bytes_per_round_per_rank": 16 * 4}))
    if mb is not None:
        mb.close(dist.barrier)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
