"""One sumcheck proof sharded over ranks (one process per GPU): the devirgo split across GPUs.

Reference: `IOPProverState::prove_batch_polys` (sumcheck/src/prover.rs:37-321) splits a virtual polynomial into
`max_thread_id` contiguous index ranges (= fixes the top log T variables), lets every thread run the first
nv - log T rounds on its range, sums the per-thread round messages through channels (prover.rs:150-170) and finishes
the last log T rounds on the merged residuals (`merge_sumcheck_polys`, util.rs:215-243).  The transcript sees
nv (total) and the degree, then one summed message per round, so the proof is byte-identical to `prove_parallel`
on the unsplit polynomial (zkml/src/model/mod.rs:987-993 asserts exactly that).

Here a "thread" is a rank.  Rank g owns elements [g*n/G, (g+1)*n/G) of every MLE, resident on its own GPU; a round is
one local device launch (dp_sc_round) plus ONE all-gather of (deg+1) Ext values (16*(deg+1) bytes per rank) -- the
only exchange the path has.  Every rank then adds the G partial messages mod p and runs the same Fiat-Shamir
transcript, so no challenge broadcast is needed (the sponge is deterministic and ~2 us per permutation on the host).
After the local rounds the G residual values per MLE are all-gathered and the last log G rounds run replicated.

The exchange is injected (`allgather`) so the same code runs over NCCL (device tensors over NVLink), over gloo
(CPU tests) or in-process; the per-slice engine is injected as well (product: the CUDA library's dp_sc_*).
"""
import ctypes as C

import numpy as np

P = 0xFFFFFFFF00000001
# the exchange callback of the sharded entry points (host/sumcheck.hpp CallbackExchange::Fn): cb(user, send, n_words, recv) -> 0 on success
_ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64))


def _sum_mod_p(parts):
    """parts: [world, k, 2] uint64 canonical -> [k, 2] uint64 (component-wise sum mod p; k is tiny: deg+1 or #MLEs)"""
    parts = np.asarray(parts, dtype=np.uint64)
    out = np.zeros(parts.shape[1:], dtype=np.uint64)
    for idx in np.ndindex(*out.shape):
        out[idx] = sum(int(parts[(g,) + idx]) for g in range(parts.shape[0])) % P
    return out


class TorchAllGather:
    """all-gather of a small uint64 array over a torch.distributed process group (NCCL: device tensors; gloo: CPU)."""

    def __init__(self, dist, device=None, group=None):
        import torch
        self.torch, self.dist, self.group = torch, dist, group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.device = device if device is not None else ("cuda" if dist.get_backend(group) == "nccl" else "cpu")

    def __call__(self, words):
        t = self.torch
        w = np.ascontiguousarray(words, dtype=np.uint64).reshape(-1)
        send = t.from_numpy(w.view(np.int64)).to(self.device)
        recv = t.empty(self.world * w.size, dtype=t.int64, device=self.device)
        self.dist.all_gather_into_tensor(recv, send, group=self.group)
        return recv.cpu().numpy().view(np.uint64).reshape(self.world, *np.shape(words))


def shard_range(n, rank, world):
    """contiguous index range owned by `rank` (the top log2(world) variables select the rank)"""
    if world & (world - 1) or n % world:
        raise ValueError("world size must be a power of two dividing the MLE length")
    per = n // world
    return rank * per, (rank + 1) * per


def prove_sharded(make_engine, local_mles, products, nv_total, max_deg, rank, world, allgather, transcript):
    """Distributed `prove_batch_polys` with max_thread_id = world.

    make_engine(mles, products, nv, max_deg) -> object with .round(challenge|None) -> [max_deg+1, 2] and
    .finish(challenge) -> [n_mles, 2]   (dpb200.Sumcheck over dpb200.Mle handles in the product);
    local_mles: this rank's slice of every MLE, in the engine's own representation;
    transcript: .append_msg(bytes) / .append_e(array[k,2]) / .challenge(label) -> [2].
    Returns (point[nv,2], msgs[nv,max_deg+1,2], final_evals[n_mles,2]) -- identical on every rank.
    """
    log_w = world.bit_length() - 1
    if world != 1 << log_w:
        raise ValueError("world size must be a power of two")
    nv_local = nv_total - log_w
    if nv_local < 1:
        raise ValueError("prove_sharded: fewer than one local variable per rank")
    transcript.append_msg(int(nv_total).to_bytes(8, "little"))      # prover.rs:70-71
    transcript.append_msg(int(max_deg).to_bytes(8, "little"))
    eng = make_engine(local_mles, products, nv_local, max_deg)
    point, msgs, ch = [], [], None
    for _ in range(nv_local):
        part = eng.round(ch)                                         # local K1/K2 launch
        msg = _sum_mod_p(allgather(part)) if world > 1 else np.asarray(part, dtype=np.uint64)
        transcript.append_e(msg)
        ch = transcript.challenge(b"Internal round")
        msgs.append(msg); point.append(ch)
    fin_local = np.asarray(eng.finish(ch), dtype=np.uint64)          # this slice's residual value of every MLE
    if world == 1:
        return np.array(point), np.array(msgs), fin_local
    residual = allgather(fin_local)                                  # [world, n_mles, 2]: merge_sumcheck_polys (util.rs:215-243)
    n_mles = residual.shape[1]
    merged = [(np.ascontiguousarray(residual[:, i, :]), True) for i in range(n_mles)]
    eng2 = make_engine(merged, products, log_w, max_deg)             # last log G rounds, replicated on every rank
    ch2 = None
    for _ in range(log_w):
        msg = np.asarray(eng2.round(ch2), dtype=np.uint64)
        transcript.append_e(msg)
        ch2 = transcript.challenge(b"Internal round")
        msgs.append(msg); point.append(ch2)
    fin = np.asarray(eng2.finish(ch2), dtype=np.uint64)
    return np.array(point), np.array(msgs), fin


# ---- product engine (CUDA library; the transcript is dpb200.Transcript of the C++ host mirror) ------------------------
def device_engine(mles, products, nv, max_deg):
    """per-slice engine on this rank's GPU: mles are dpb200.Mle handles, or (array, is_ext) pairs that get uploaded"""
    import dpb200 as dp
    hs = [m if isinstance(m, dp.Mle) else dp.Mle.upload(m[0], m[1]) for m in mles]
    return dp.Sumcheck(hs, products, nv, max_deg)


def prove_sharded_device(local_mles, products, nv_total, rank, world, allgather, label=b"m2vec"):
    """the product entry: this rank's slices are resident on its GPU (dp_init done by the caller)"""
    import dpb200 as dp
    max_deg = max(len(p[1]) for p in products)
    return prove_sharded(device_engine, local_mles, products, nv_total, max_deg, rank, world, allgather, dp.Transcript(label))


# ---- native path: the whole sharded proof inside the C++ host mirror, exchange through shared memory -----------
def _exchange_args(mailbox, allgather, world):
    """the (shm_region, shm_seq, cb, user) arguments of a sharded entry point: the mailbox, or a callback over `allgather` (keep the
    tuple until the call returns: it holds the callback)."""
    if mailbox is not None:
        return C.c_void_p(mailbox.addr), C.byref(mailbox.seq), None, None
    if allgather is None:
        return None, None, None, None

    def cb(user, send, n, recv):
        try:
            got = allgather(np.ctypeslib.as_array(send, shape=(int(n),)).copy())
            np.ctypeslib.as_array(recv, shape=(world * int(n),))[:] = np.asarray(got, dtype=np.uint64).reshape(-1)
            return 0
        except Exception:
            return 1
    return None, None, _ALLGATHER_FN(cb), None


class ShmMailbox:
    """Same-node mailbox for IOPProverState::prove_sharded (host/sumcheck.hpp ShmExchange): one zero-initialised POSIX
    shared-memory region mapped by every rank.  The per-round message must reach the host for Fiat-Shamir anyway, so
    the ranks exchange it host-to-host (~1 us) instead of through a device collective."""

    def __init__(self, name, rank, world, barrier):
        from multiprocessing import shared_memory, resource_tracker
        import dpb200 as dp
        size = int(dp.host().dph_shm_mailbox_bytes())
        self.rank, self.world = rank, world
        if rank == 0:
            self.shm = shared_memory.SharedMemory(name=name, create=True, size=size)
            self.shm.buf[:size] = bytes(size)
        barrier()
        if rank != 0:
            self.shm = shared_memory.SharedMemory(name=name)
            try:
                resource_tracker.unregister(self.shm._name, "shared_memory")   # rank 0 owns the segment
            except Exception:
                pass
        barrier()
        self._anchor = C.c_char.from_buffer(self.shm.buf)
        self.addr = C.addressof(self._anchor)
        self.seq = C.c_uint64(0)

    def close(self, barrier=None):
        del self._anchor
        if barrier is not None:
            barrier()
        self.shm.close()
        if self.rank == 0:
            self.shm.unlink()


def prove_sharded_native(local_mles, products, nv_total, rank, world, mailbox=None, allgather=None, label=b"m2vec"):
    """IOPProverState::prove_sharded in the C++ host mirror (no Python in the round loop).  Exchange: `mailbox`
    (ShmMailbox, same node) or `allgather` (callable(words)->[world, n], e.g. TorchAllGather over NCCL)."""
    import dpb200 as dp
    prods = dp.make_products(products)
    max_deg = max(len(p[1]) for p in products)
    point = np.zeros((nv_total, 2), dtype=np.uint64)
    msgs = np.zeros((nv_total, max_deg + 1, 2), dtype=np.uint64)
    fin = np.zeros((len(local_mles), 2), dtype=np.uint64)
    ex = _exchange_args(mailbox, allgather, world)
    dp.hcheck(dp.host().dph_sumcheck_prove_sharded(world, rank, dp.handles(local_mles), len(local_mles), prods, len(products), nv_total, label,
                                                   *ex, point.ctypes.data, msgs.ctypes.data, fin.ctypes.data))
    return point, msgs, fin


# ---- Basefold commit + open of ONE polynomial sharded over the ranks (BASELINE configs[3]: 2^24 evaluations, 1 vs 8 GPUs) --------
class LocalMailbox:
    """The ShmExchange mailbox in plain process memory: `world` threads of ONE process (each with its own library context on the
    same GPU) can play the ranks -- how the single-GPU tests exercise the sharded protocol end to end."""

    def __init__(self):
        import dpb200 as dp
        self.buf = (C.c_char * int(dp.host().dph_shm_mailbox_bytes()))()
        self.addr = C.addressof(self.buf)

    def for_rank(self):
        class _View:
            pass
        v = _View(); v.addr = self.addr; v.seq = C.c_uint64(0)
        return v


def basefold_commit_open_sharded(mle, full_log, point, rank, world, mailbox=None, allgather=None, label=b"m2vec", cap=1 << 24):
    """Basefold::commit_sharded + open_sharded of the C++ host mirror (host/mpcs.hpp): `mle` is the WHOLE polynomial resident on
    this rank's GPU; this rank keeps the slice [rank/world, (rank+1)/world) of the bit-reversed evaluations, codeword, oracles and
    Merkle trees.  Exchange: `mailbox` (ShmMailbox / LocalMailbox view) or `allgather` (callable(words) -> [world, n]).
    Returns (root[4], flat proof (same image as dpb200.pcs_open), (commit_ms, open_ms)) -- identical on every rank."""
    import dpb200 as dp
    p = np.ascontiguousarray(point, dtype=np.uint64).reshape(-1)
    root, times = np.zeros(4, dtype=np.uint64), np.zeros(2, dtype=np.float64)
    ex = _exchange_args(mailbox, allgather, world)
    flat = dp.flat_out(cap, lambda *o: dp.host().dph_pcs_open_sharded(world, rank, mle.h, full_log, p.ctypes.data, label, *ex, *o,
                                                                      root.ctypes.data, times.ctypes.data))
    return root, flat, (float(times[0]), float(times[1]))
