"""N>1 host logic on CPU (gloo, world_size 2): the replica arm's max-over-ranks timing / whole-job value, and the
reference arm's "rank 0 alone works and prints, other ranks exit 0" rule (task statement sections 4 and 5)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import os, sys, json
sys.path.insert(0, %r)
import torch, torch.distributed as dist
import bench
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
ms = 10.0 + 5.0 * rank                       # rank 1 is slower
agg = bench.max_over_ranks(ms, dist, device="cpu")
val = bench.whole_job_value(4, world, agg)
dist.barrier()
if rank == 0:
    print(json.dumps({"agg_ms": agg, "value": val, "world": world}))
dist.destroy_process_group()
''' % ROOT


def _torchrun(args, timeout=300, nproc=2):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
           "--master-port", str(29613 + nproc)] + args
    return subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env, cwd=ROOT)


def test_replica_timing_is_max_over_ranks(tmp_path):
    w = tmp_path / "worker.py"
    w.write_text(WORKER)
    r = _torchrun([str(w)])
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(line) == 1
    out = json.loads(line[0])
    assert out["world"] == 2 and out["agg_ms"] == 15.0           # the slower rank
    assert abs(out["value"] - 8 / 0.015) < 1e-6                   # 2 ranks x 4 proofs / 15 ms


def test_reference_arm_under_torchrun_prints_once():
    r = _torchrun(["bench.py", "--impl", "reference", "--workload", "sumcheck20", "--only", "--gpus", "2", "--steps", "1", "--warmup", "0"])   # --only: the other workloads' CPU arms take minutes on a small box
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout
    out = json.loads(lines[0])
    assert out["impl"] == "reference" and out["n_gpus"] == 2 and out["cpu_baseline"]["kind"] == "port"
    assert out["e2e"]["h2d_bytes_per_step"] == 0 and out["value"] > 0


SHARDED_WORKER = r'''
import os, sys, json
import numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests")); sys.path.insert(0, os.path.join(%(root)r, "deep-prove_b200"))
import torch, torch.distributed as dist
import oracle_py as O
import multigpu as mg

class OracleSliceEngine:
    """CPU stand-in for dp_sc_* on one slice (tests only): recomputes the round message from the challenge prefix"""
    def __init__(self, mles, products, nv, max_deg):
        self.mles, self.products, self.nv, self.ch = mles, products, nv, []
    def _run(self):
        ch = np.zeros((self.nv, 2), dtype=np.uint64)
        for i, c in enumerate(self.ch): ch[i] = c
        return O.sumcheck_rounds_fixed(self.mles, self.products, self.nv, ch)
    def round(self, c):
        if c is not None: self.ch.append(np.asarray(c, dtype=np.uint64))
        return self._run()[0][len(self.ch)]
    def finish(self, c):
        self.ch.append(np.asarray(c, dtype=np.uint64))
        return self._run()[1]

dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
nv = 9
full = [(O.splitmix_f(11, 1 << nv), False), (O.splitmix_e(12, 1 << nv), True), (O.splitmix_f(13, 1 << nv), False)]
products = [((1, 0), [0, 1, 2]), ((5, 7), [1, 2])]
lo, hi = mg.shard_range(1 << nv, rank, world)
local = [((a.reshape(-1, 2)[lo:hi] if e else a[lo:hi]).copy(), e) for a, e in full]
point, msgs, fin = mg.prove_sharded(OracleSliceEngine, local, products, nv, 3, rank, world, mg.TorchAllGather(dist), O.Transcript(b"m2vec"))
ep, em, ef = O.sumcheck_prove(full, products, nv)
ok = bool((point == ep).all() and (msgs == em).all() and (fin == ef).all())
flags = [None] * world
dist.all_gather_object(flags, ok)
if rank == 0:
    print(json.dumps({"ok": all(flags), "world": world, "rounds": int(msgs.shape[0])}))
dist.destroy_process_group()
'''


import pytest  # noqa: E402


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_sumcheck_equals_unsplit_proof(tmp_path, world):
    """devirgo split across ranks (multigpu.prove_sharded) == prove_parallel on the unsplit polynomial, on every rank
    (the identity zkml/src/model/mod.rs:987-993 asserts); exchange over gloo, slices evaluated by the CPU checker"""
    w = tmp_path / "sharded.py"
    w.write_text(SHARDED_WORKER % {"root": ROOT})
    r = _torchrun([str(w)], nproc=world)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][0])
    assert out == {"ok": True, "world": world, "rounds": 9}


SHM_WORKER = r'''
import os, sys, json, ctypes as C
import numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "deep-prove_b200"))
import torch.distributed as dist
import dpb200 as dp, multigpu as mg
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
mb = mg.ShmMailbox("dpb200_cpu_%%d" %% os.getppid(), rank, world, dist.barrier)
H = dp.host()
ok = True
for it in range(2000):
    n = [8, 1, 2046, 2047, 5000][it %% 5]         # one slot, a full slot, and multi-chunk payloads (the sharded Basefold query rows)
    send = (np.arange(n, dtype=np.uint64) * np.uint64(1000003) + np.uint64(it * 17 + rank)).astype(np.uint64)
    recv = np.zeros(world * n, dtype=np.uint64)
    assert H.dph_shm_allgather(C.c_void_p(mb.addr), world, rank, C.byref(mb.seq), send.ctypes.data, n, recv.ctypes.data) == 0
    for g in range(world):
        exp = (np.arange(n, dtype=np.uint64) * np.uint64(1000003) + np.uint64(it * 17 + g)).astype(np.uint64)
        ok = ok and bool((recv[g * n:(g + 1) * n] == exp).all())
flags = [None] * world
dist.all_gather_object(flags, ok)
mb.close(dist.barrier)
if rank == 0:
    print(json.dumps({"ok": all(flags), "seq": int(mb.seq.value)}))
dist.destroy_process_group()
'''


def test_shared_memory_mailbox_allgather(tmp_path):
    """the same-node exchange used by prove_sharded (host/sumcheck.hpp ShmExchange): 2000 back-to-back all-gathers
    between two processes, including payloads larger than one slot"""
    w = tmp_path / "shm.py"
    w.write_text(SHM_WORKER % {"root": ROOT})
    r = _torchrun([str(w)])
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][0])
    assert out["ok"] is True and out["seq"] == 400 * (1 + 1 + 1 + 2 + 3)
