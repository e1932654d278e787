// Context, error reporting, device arena and pinned-memory plumbing of libdeepprove_b200.so.
#include "common.cuh"
#include <cstdlib>
#include <atomic>
#include <mutex>

static thread_local std::string g_err;
// One context PER HOST THREAD (own stream, device arena, pinned cache): independent proofs run concurrently
// from several host threads on one GPU and share only read-only device data (model, tables, twiddles).  Only the owning thread
// reaches its context, so nothing in it is locked.
static thread_local DpCtx g_ctx;
DpCtx &dp_ctx() { return g_ctx; }
static std::atomic<unsigned long long> g_total_launches{0};
void dp_count_launch() { g_total_launches.fetch_add(1, std::memory_order_relaxed); }
static std::atomic<unsigned long long> g_host_waits{0};
int dp_fail(int code, const std::string &s) { g_err = s; return code; }

// ---- per-thread device arena -------------------------------------------------------------------------
// A proof makes thousands of short-lived allocations (ping-pong tables, eq tables, partials).  Going to the
// driver for each one (even cudaMallocAsync) serialises concurrent proving threads on driver locks, so each
// context sub-allocates from big cudaMalloc'ed slabs with power-of-two size classes on the host.  All work of a
// context is ordered on its one stream, so a block may be reused as soon as it is released; the only
// multi-stream section (dp_pcs_commit_many) defers its releases until its streams have been joined.
#include <unordered_map>
struct DpArena {
    struct Slab { char *base; size_t cap, used; };
    std::vector<Slab> slabs;
    std::vector<void *> free_list[48];
    std::unordered_map<void *, unsigned char> cls;
    std::vector<void *> deferred; bool defer = false;
    // blocks of THIS arena released by other host threads (e.g. a handle created on one proving thread and destroyed on
    // another): parked here under the registry lock and folded back into the free lists by the owner's next allocation
    std::vector<void *> returned; std::atomic<unsigned> n_returned{0};
    ~DpArena();
};
// process-wide slab registry: which arena owns an address (only consulted on the rare foreign free and on teardown)
struct SlabReg { char *base; size_t cap; DpArena *owner; };
static std::vector<SlabReg> g_slab_reg;
static std::mutex g_slab_mu;
static thread_local DpArena g_arena;
static constexpr size_t ARENA_SLAB = 256ull << 20;
static void arena_release_slabs(DpArena &a) {
    {
        std::lock_guard<std::mutex> lk(g_slab_mu);
        for (size_t i = 0; i < g_slab_reg.size();) { if (g_slab_reg[i].owner == &a) { g_slab_reg[i] = g_slab_reg.back(); g_slab_reg.pop_back(); } else i++; }
        a.returned.clear(); a.n_returned = 0;
    }
    for (auto &s : a.slabs) cudaFree(s.base);    // after the runtime has shut down this is a harmless error
    a.slabs.clear();
}
// a host thread that exits without dp_shutdown() must not leak its >= 256 MB slabs
DpArena::~DpArena() { arena_release_slabs(*this); }
void dp_arena_defer(bool on) {
    g_arena.defer = on;
    if (!on) { for (void *p : g_arena.deferred) { auto it = g_arena.cls.find(p); if (it != g_arena.cls.end()) g_arena.free_list[it->second].push_back(p); } g_arena.deferred.clear(); }
}
static void arena_drain_returned(DpArena &a) {
    std::lock_guard<std::mutex> lk(g_slab_mu);
    for (void *p : a.returned) { auto it = a.cls.find(p); if (it != a.cls.end()) a.free_list[it->second].push_back(p); }
    a.returned.clear(); a.n_returned = 0;
}
int dp_dev_alloc(void **p, size_t bytes) {
    if (bytes < 256) bytes = 256;
    unsigned c = 8; while (((size_t)1 << c) < bytes) c++;
    DpArena &a = g_arena;
    if (a.free_list[c].empty() && a.n_returned.load(std::memory_order_acquire)) arena_drain_returned(a);
    if (!a.free_list[c].empty()) { *p = a.free_list[c].back(); a.free_list[c].pop_back(); return DP_OK; }
    size_t need = (size_t)1 << c;
    for (auto &s : a.slabs) if (s.cap - s.used >= need) { *p = s.base + s.used; s.used += need; a.cls[*p] = (unsigned char)c; return DP_OK; }
    size_t cap = need > ARENA_SLAB ? need : ARENA_SLAB;
    char *base = nullptr;
    DP_CUDA(cudaMalloc((void **)&base, cap));
    a.slabs.push_back({base, cap, need});
    { std::lock_guard<std::mutex> lk(g_slab_mu); g_slab_reg.push_back({base, cap, &a}); }
    *p = base; a.cls[*p] = (unsigned char)c;
    return DP_OK;
}
int dp_dev_free(void *p) {
    if (!p) return DP_OK;
    DpArena &a = g_arena;
    auto it = a.cls.find(p);
    if (it == a.cls.end()) {
        // owned by another thread's arena: hand it back to its owner.  The owner's stream knows nothing about the work this
        // thread queued on the block, so that work is drained first (foreign frees are rare: cross-thread handle teardown).
        if (g_ctx.ready && g_ctx.stream) cudaStreamSynchronize(g_ctx.stream);
        std::lock_guard<std::mutex> lk(g_slab_mu);
        for (auto &r : g_slab_reg) if ((char *)p >= r.base && (char *)p < r.base + r.cap) { r.owner->returned.push_back(p); r.owner->n_returned.fetch_add(1, std::memory_order_release); break; }
        return DP_OK;
    }
    if (a.defer) a.deferred.push_back(p); else a.free_list[it->second].push_back(p);
    return DP_OK;
}
static void arena_destroy() {
    arena_release_slabs(g_arena);
    for (auto &f : g_arena.free_list) f.clear();
    g_arena.cls.clear(); g_arena.deferred.clear(); g_arena.defer = false;
}

// Pinned (mapped) host blocks: power-of-two size classes, a 64-byte header in front of every block holds its class, free blocks sit
// in a PER-THREAD cache (no lock, O(1)); a process-wide pool takes the caches of threads that exit and serves cache misses before the
// driver is asked (cudaHostAlloc costs ~ms and synchronises the device: never on the proving path once warm).  The first version
// kept one process-wide list under a mutex and scanned it linearly on every alloc and free: with 48 proving threads and thousands
// of blocks that made dp_sc_create / dp_sc_destroy a large share of a Dense-4M proof's host CPU time.
static constexpr int PIN_CLASSES = 40;
struct PinnedPool { std::mutex mu; std::vector<void *> free_[PIN_CLASSES]; };
static PinnedPool g_pin_pool;
struct PinnedCache {
    std::vector<void *> free_[PIN_CLASSES];
    ~PinnedCache() { std::lock_guard<std::mutex> lk(g_pin_pool.mu); for (int c = 0; c < PIN_CLASSES; c++) for (void *p : free_[c]) g_pin_pool.free_[c].push_back(p); }
};
static thread_local PinnedCache g_pin_cache;
int dp_pinned_alloc(void **p, size_t bytes) {
    int c = 12; while (((size_t)1 << c) < bytes) c++;            // 4 KiB minimum, as before
    if (c >= PIN_CLASSES) return dp_fail(DP_ERR_INVALID, "dp_pinned_alloc: request too large");
    auto &mine = g_pin_cache.free_[c];
    if (!mine.empty()) { *p = mine.back(); mine.pop_back(); return DP_OK; }
    {
        std::lock_guard<std::mutex> lk(g_pin_pool.mu);
        auto &pool = g_pin_pool.free_[c];
        if (!pool.empty()) { *p = pool.back(); pool.pop_back(); return DP_OK; }
    }
    char *q = nullptr;
    DP_CUDA(cudaHostAlloc((void **)&q, ((size_t)1 << c) + 64, cudaHostAllocMapped));   // device-visible: kernels read descriptors / write results in place
    *(int *)q = c;
    *p = q + 64;
    return DP_OK;
}
void dp_pinned_free(void *p) {
    if (!p) return;
    const int c = *(const int *)((const char *)p - 64);
    if (c < 12 || c >= PIN_CLASSES) return;      // not one of ours
    g_pin_cache.free_[c].push_back(p);
}

#include <chrono>
// ---- waiting without burning a core (see common.cuh) -------------------------------------------------------------------
#include <thread>
#include <linux/futex.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <time.h>
static std::atomic<int> g_wait_mode{DP_WAIT_SPIN};
int dp_wait_mode() { return g_wait_mode.load(std::memory_order_relaxed); }
static long futex_call(std::atomic<u32> *addr, int op, u32 val, const struct timespec *ts) { return syscall(SYS_futex, (u32 *)addr, op, val, ts, nullptr, 0); }
struct WaitSlot {
    std::atomic<u32> state{0};                 // 0 idle, 1 armed (the poller watches it), 3 being fired by the poller, 2 fired
    volatile u64 *flag = nullptr; u64 want = 0, fail = 0; bool has_fail = false;
    u64 seen = 0;
    std::atomic<u32> wake{0};                  // futex word the owner sleeps on
    char pad[64];
};
static constexpr u32 WAIT_SLOTS = 1024;
static WaitSlot g_wslots[WAIT_SLOTS];
static std::atomic<u32> g_wslots_used{0}, g_armed{0}, g_poller_gen{0};
static std::once_flag g_poller_once;
static void poller_main() {
    for (;;) {
        if (g_armed.load(std::memory_order_acquire) == 0) {       // nothing to watch: sleep until a waiter arms a slot
            const u32 gen = g_poller_gen.load(std::memory_order_acquire);
            if (g_armed.load(std::memory_order_acquire) == 0) { struct timespec ts = {0, 2000000}; futex_call(&g_poller_gen, FUTEX_WAIT_PRIVATE, gen, &ts); }
            continue;
        }
        const u32 n = std::min<u32>(g_wslots_used.load(std::memory_order_acquire), WAIT_SLOTS);
        for (u32 i = 0; i < n; i++) {
            WaitSlot &w = g_wslots[i];
            if (w.state.load(std::memory_order_acquire) != 1) continue;
            const u64 v = *w.flag;
            if (v == w.want || (w.has_fail && v == w.fail)) {
                u32 armed = 1;                               // claim the slot first: a waiter that is timing out withdraws it with the same CAS
                if (!w.state.compare_exchange_strong(armed, 3, std::memory_order_acq_rel)) continue;
                w.seen = v;
                g_armed.fetch_sub(1, std::memory_order_acq_rel);
                w.state.store(2, std::memory_order_release);
                w.wake.store(1, std::memory_order_release);
                futex_call(&w.wake, FUTEX_WAKE_PRIVATE, 1, nullptr);
            }
        }
        __builtin_ia32_pause();
    }
}
u64 dp_wait_flag(volatile u64 *flag, u64 want, bool has_fail, u64 fail, double timeout_s) {
    g_host_waits.fetch_add(1, std::memory_order_relaxed);
    // a result that is already there (or lands within a microsecond) never pays for a sleep
    for (int k = 0; k < 64; k++) { const u64 v = *flag; if (v == want || (has_fail && v == fail)) return v; __builtin_ia32_pause(); }
    const auto t_start = std::chrono::steady_clock::now();
    if (dp_wait_mode() == DP_WAIT_SPIN) {
        for (u64 spins = 1;; spins++) {
            const u64 v = *flag; if (v == want || (has_fail && v == fail)) return v;
            if ((spins & 0xFFFF) == 0 && std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count() > timeout_s) return DP_WAIT_TIMEOUT;
            __builtin_ia32_pause();
        }
    }
    // BLOCK mode: a bounded number of waiters may still spin for a short while (lowest latency for the proofs that are in
    // their round-trip-bound phases) -- never more than about half of the CPUs this process may use.
    {
        static const int spin_limit = [] {
            double cpus = (double)std::thread::hardware_concurrency();
            if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) { char q[64]; double per = 0; if (fscanf(f, "%63s %lf", q, &per) == 2 && strcmp(q, "max") != 0 && per > 0) cpus = std::min(cpus, atof(q) / per); fclose(f); }
            // one process per GPU on a shared box (torchrun): this process's share of the CPUs, not the whole container's
            if (const char *lw = getenv("LOCAL_WORLD_SIZE")) { const int w = atoi(lw); if (w > 1) cpus /= w; }
            return std::max(0, (int)(cpus / 2) - 2);
        }();
        static std::atomic<int> spinners{0};
        if (spin_limit > 0 && spinners.fetch_add(1, std::memory_order_acq_rel) < spin_limit) {
            u64 seen = DP_WAIT_TIMEOUT; bool got = false;
            for (u64 spins = 1;; spins++) {
                const u64 v = *flag; if (v == want || (has_fail && v == fail)) { seen = v; got = true; break; }
                if ((spins & 0x3FF) == 0 && std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count() > 60e-6) break;
                __builtin_ia32_pause();
            }
            spinners.fetch_sub(1, std::memory_order_acq_rel);
            if (got) return seen;
        } else spinners.fetch_sub(1, std::memory_order_acq_rel);
    }
    static thread_local int my_slot = -1;
    if (my_slot < 0) {
        const u32 idx = g_wslots_used.fetch_add(1, std::memory_order_acq_rel);
        if (idx >= WAIT_SLOTS) { g_wslots_used.store(WAIT_SLOTS); my_slot = -2; } else my_slot = (int)idx;
    }
    if (my_slot == -2) {   // more waiting threads than slots (never in practice): sleep-poll
        for (;;) {
            const u64 v = *flag; if (v == want || (has_fail && v == fail)) return v;
            if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count() > timeout_s) return DP_WAIT_TIMEOUT;
            struct timespec ts = {0, 20000}; nanosleep(&ts, nullptr);
        }
    }
    std::call_once(g_poller_once, [] { std::thread(poller_main).detach(); });
    WaitSlot &w = g_wslots[my_slot];
    w.flag = flag; w.want = want; w.fail = fail; w.has_fail = has_fail; w.wake.store(0, std::memory_order_relaxed);
    const u32 armed_before = g_armed.fetch_add(1, std::memory_order_acq_rel);
    w.state.store(1, std::memory_order_release);
    if (armed_before == 0) { g_poller_gen.fetch_add(1, std::memory_order_acq_rel); futex_call(&g_poller_gen, FUTEX_WAKE_PRIVATE, 1, nullptr); }
    for (;;) {
        if (w.wake.load(std::memory_order_acquire) == 0) { struct timespec ts = {0, 5000000}; futex_call(&w.wake, FUTEX_WAIT_PRIVATE, 0, &ts); }
        if (w.state.load(std::memory_order_acquire) == 2) { const u64 v = w.seen; w.state.store(0, std::memory_order_release); return v; }
        if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count() > timeout_s) {
            // withdraw the slot; if the poller fires it at this very moment the result is simply taken
            u32 one = 1;
            if (w.state.compare_exchange_strong(one, 0, std::memory_order_acq_rel)) { g_armed.fetch_sub(1, std::memory_order_acq_rel); return DP_WAIT_TIMEOUT; }
        }
    }
}
__global__ void k_signal(u64 *flag, u64 seq) { dp_publish(flag, seq); }
cudaError_t dp_stream_sync(cudaStream_t st) {
    if (dp_wait_mode() == DP_WAIT_SPIN) { g_host_waits.fetch_add(1, std::memory_order_relaxed); return cudaStreamSynchronize(st); }
    DpCtx &c = g_ctx;
    if (!c.sync_flag) { void *p = nullptr; if (dp_pinned_alloc(&p, 64) != DP_OK) return cudaErrorMemoryAllocation; c.sync_flag = (u64 *)p; *c.sync_flag = 0; c.sync_seq = 0; }
    const u64 seq = ++c.sync_seq;
    if (cudaError_t e = dp_launch(k_signal, 1, 1, 0, st, c.sync_flag, seq)) return e;
    if (dp_wait_flag(c.sync_flag, seq, false, 0, 30.0) != seq) return cudaStreamSynchronize(st);   // timeout: let the runtime report what happened
    return cudaSuccess;
}
int dp_await(volatile u64 *word, u64 want, double timeout_s, const std::string &refusal) {
    if (dp_wait_flag(word, want, false, 0, timeout_s) == want) return DP_OK;
    DP_CUDA(dp_stream_sync(g_ctx.stream));
    DP_CHECK(*word == want, DP_ERR_CUDA, refusal);
    return DP_OK;
}

DpD2H::DpD2H(cudaStream_t s, size_t reserve_bytes) : st(s) { cap = reserve_bytes < 64 ? 64 : reserve_bytes; if (dp_pinned_alloc(&pin, cap) != DP_OK) { pin = nullptr; cap = 0; } }
DpD2H::~DpD2H() { if (!pieces.empty()) cudaStreamSynchronize(st); dp_pinned_free(pin); }   // copies still in flight (an error path skipped finish()): the block must not be recycled under them
int DpD2H::add(void *host_dst, const void *dev_src, size_t bytes) {
    if (!pin || used + bytes > cap) return dp_fail(DP_ERR_CUDA, "DpD2H: staging buffer too small or not allocated");
    DP_CUDA(cudaMemcpyAsync((char *)pin + used, dev_src, bytes, cudaMemcpyDeviceToHost, st));
    pieces.push_back({host_dst, used, bytes});
    used += (bytes + 15) & ~(size_t)15;
    return DP_OK;
}
int DpD2H::finish() {
    DP_CUDA(dp_stream_sync(st));
    for (auto &p : pieces) memcpy(p.dst, (char *)pin + p.off, p.bytes);
    pieces.clear(); used = 0;
    return DP_OK;
}
int dp_d2h(void *host_dst, const void *dev_src, size_t bytes, cudaStream_t st) {
    DpD2H x(st, bytes);
    if (int e = x.add(host_dst, dev_src, bytes)) return e;
    return x.finish();
}

int dp_zero_block_get(void **p) {
    DpCtx &c = g_ctx;
    if (!c.zero_blocks.empty()) { *p = c.zero_blocks.back(); c.zero_blocks.pop_back(); return DP_OK; }
    if (int e = dp_dev_alloc(p, 256)) return e;
    DP_CUDA(cudaMemsetAsync(*p, 0, 256, c.stream));
    return DP_OK;
}
void dp_zero_block_put(void *p) { if (p) g_ctx.zero_blocks.push_back(p); }

// ---- per-kernel event timing --------------------------------------------------------------------
// Process-wide switch and statistics, thread-local event lists: every proving thread brackets its launches with events
// on ITS stream and folds the elapsed times into the shared table (dp_profile_flush at the end of a proof, or any
// dp_profile_* call), so a batch of concurrent proofs yields the per-kernel breakdown of the concurrent region itself.
#include <map>
struct ProfRec { cudaEvent_t a, b; std::string name; u64 bytes, units; };
struct ProfStat { u64 count = 0; double ms = 0; u64 bytes = 0, units = 0; };
static std::atomic<bool> g_prof_on{false};
static thread_local std::vector<ProfRec> g_prof_pending;
static thread_local std::vector<cudaEvent_t> g_prof_pool;
static std::map<std::string, ProfStat> g_prof_stats;
static std::mutex g_prof_mu;
static cudaEvent_t prof_event() {
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
}
int dp_prof_begin(const char *name, u64 bytes, u64 units) {
    if (!g_prof_on.load(std::memory_order_relaxed)) return -1;
    ProfRec r; r.a = prof_event(); r.b = prof_event(); r.name = name; r.bytes = bytes; r.units = units;
    cudaEventRecord(r.a, g_ctx.stream);
    g_prof_pending.push_back(r);
    return (int)g_prof_pending.size() - 1;
}
void dp_prof_end(int tok) { if (tok >= 0 && tok < (int)g_prof_pending.size()) cudaEventRecord(g_prof_pending[tok].b, g_ctx.stream); }
static void prof_resolve() {
    if (g_prof_pending.empty()) return;
    cudaStreamSynchronize(g_ctx.stream);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (auto &r : g_prof_pending) {
        float ms = 0; cudaEventElapsedTime(&ms, r.a, r.b);
        ProfStat &s = g_prof_stats[r.name]; s.count++; s.ms += ms; s.bytes += r.bytes; s.units += r.units;
        g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b);
    }
    g_prof_pending.clear();
}

extern "C" {

// test hook (not part of the ABI): the wait service on an arbitrary word -- lets the CPU suite exercise the poller / futex path without a device
uint64_t dp_debug_wait_flag(volatile uint64_t *flag, uint64_t want, double timeout_s) { return dp_wait_flag((volatile u64 *)flag, want, false, 0, timeout_s); }

int dp_set_wait_mode(int mode) {
    if (mode != DP_WAIT_SPIN && mode != DP_WAIT_BLOCK) return dp_fail(DP_ERR_INVALID, "dp_set_wait_mode: 0 = spin, 1 = block on the poller thread");
    g_wait_mode.store(mode);
    return DP_OK;
}
int dp_get_wait_mode(void) { return dp_wait_mode(); }

int dp_profile_enable(int on) {
    prof_resolve();
    g_prof_on.store(on != 0);
    return DP_OK;
}
int dp_profile_flush(void) {   // fold this thread's pending events into the process-wide table (cheap no-op when idle)
    if (g_prof_pending.empty()) return DP_OK;
    prof_resolve();
    return DP_OK;
}
int dp_profile_reset(void) {
    prof_resolve();
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_stats.clear();
    return DP_OK;
}
// Writes up to `cap` entries; returns the number of distinct kernel names seen.  `units` (may be NULL) = the kernel's own
// work unit summed over launches: Poseidon2 permutations for the Merkle kernels, field operations for the sumcheck rounds.
int dp_profile_read_ex(char (*names)[64], uint64_t *counts, double *total_ms, uint64_t *bytes, uint64_t *units, int cap) {
    prof_resolve();
    std::lock_guard<std::mutex> lk(g_prof_mu);
    int i = 0;
    for (auto &kv : g_prof_stats) {
        if (i < cap) {
            snprintf(names[i], 64, "%s", kv.first.c_str());
            counts[i] = kv.second.count; total_ms[i] = kv.second.ms; bytes[i] = kv.second.bytes;
            if (units) units[i] = kv.second.units;
        }
        i++;
    }
    return i;
}

const char *dp_last_error(void) { return g_err.c_str(); }
const char *dp_version(void) { return "deepprove_b200 0.1 (sm_90a)"; }

int dp_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int dp_init(int device) {
    // many small kernels from many streams: the default of 8 hardware work queues makes unrelated streams wait on each
    // other (a resident tail kernel in a shared queue stalls its neighbours); 32 is the hardware maximum.  Only effective
    // if CUDA is not initialised yet in this process -- hosts that initialise CUDA first should export it themselves.
    setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
    int n = dp_device_count();
    if (n <= 0) return dp_fail(DP_ERR_NO_DEVICE, "no CUDA device visible: deepprove_b200 has no CPU fallback");
    if (device < 0 || device >= n) return dp_fail(DP_ERR_INVALID, "dp_init: device index out of range");
    DP_CUDA(cudaSetDevice(device));
    if (g_ctx.ready && g_ctx.device == device) return DP_OK;
    // the stream and the arena of this thread's context belong to the device it was initialised on
    if (g_ctx.ready) { cudaSetDevice(g_ctx.device); return dp_fail(DP_ERR_STATE, "dp_init: this thread's context is bound to another device; call dp_shutdown() first"); }
    cudaDeviceProp prop;
    DP_CUDA(cudaGetDeviceProperties(&prop, device));
    g_ctx.sm_count = prop.multiProcessorCount;
    if (!g_ctx.stream) { DP_CUDA(cudaStreamCreateWithFlags(&g_ctx.stream, cudaStreamNonBlocking)); g_ctx.own_stream = true; }
    g_ctx.device = device;
    g_ctx.ready = true;
    return DP_OK;
}

int dp_shutdown(void) {
    if (!g_ctx.ready) return DP_OK;
    cudaStreamSynchronize(g_ctx.stream);
    if (g_ctx.own_stream) cudaStreamDestroy(g_ctx.stream);
    g_ctx.stream = nullptr; g_ctx.own_stream = false; g_ctx.ready = false;
    if (g_ctx.sync_flag) { dp_pinned_free(g_ctx.sync_flag); g_ctx.sync_flag = nullptr; }
    g_ctx.zero_blocks.clear();     // they live in the arena that is released below
    arena_destroy();
    return DP_OK;
}

int dp_set_stream(void *s) {
    DP_REQUIRE_CTX();
    DP_CUDA(cudaStreamSynchronize(g_ctx.stream));
    if (g_ctx.own_stream) { cudaStreamDestroy(g_ctx.stream); g_ctx.own_stream = false; }
    g_ctx.stream = (cudaStream_t)s;
    return DP_OK;
}

int dp_synchronize(void) {
    DP_REQUIRE_CTX();
    DP_CUDA(cudaStreamSynchronize(g_ctx.stream));
    return DP_OK;
}

// launches of the calling thread's context + those folded in by threads that have shut down
uint64_t dp_kernel_launches(void) { return g_total_launches.load(); }   // process-wide, all host threads
uint64_t dp_host_waits(void) { return g_host_waits.load(); }             // process-wide, all host threads

}  // extern "C"
