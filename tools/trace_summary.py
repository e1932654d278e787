#!/usr/bin/env python3
"""Summarise a CUPTI kernel timeline (tools/cupti_trace.cpp): per kernel class count / mean duration / share of GPU-resident
block-time, GPU busy fraction, and how much of the machine's thread slots and registers the running kernels hold over time."""
import csv, re, sys, collections
SM, THREADS_PER_SM, REGS_PER_SM = 132, 2048, 65536

def short(n):
    n = re.sub(r"^_Z\d+", "", n)
    m = re.match(r"(k_[a-z0-9_]+)", n)
    return m.group(1) if m else n[:24]

def main(path):
    rows = []
    for r in csv.DictReader(open(path)):
        rows.append((short(r["name"]), int(r["start_ns"]), int(r["end_ns"]), int(r["grid"]), int(r["block"]), int(r["regs"]), int(r["smem"]), int(r["stream"])))
    if not rows:
        print("no records"); return
    t0 = min(r[1] for r in rows); t1 = max(r[2] for r in rows); span = (t1 - t0) / 1e3
    print("records %d, span %.1f ms, streams %d" % (len(rows), span / 1e3, len(set(r[7] for r in rows))))
    agg = collections.defaultdict(lambda: [0, 0.0, 0.0, 0.0, 0])
    for n, s, e, g, b, rg, sm, st in rows:
        d = (e - s) / 1e3
        a = agg[n]; a[0] += 1; a[1] += d
        # capacity the kernel may hold while it runs: min(grid, what fits) blocks
        per_sm = max(1, min(THREADS_PER_SM // max(b, 1), REGS_PER_SM // max(1, rg * b)))
        resident = min(g, per_sm * SM)
        a[2] += d * resident * b / (SM * THREADS_PER_SM)           # thread-slot fraction x time
        a[3] += d * resident * b * rg / (SM * REGS_PER_SM)         # register fraction x time
        a[4] = max(a[4], g)
    print("%-22s %7s %10s %9s %12s %12s %9s" % ("kernel", "n", "sum ms", "mean us", "thr-slot ms", "reg-file ms", "max grid"))
    for n, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("%-22s %7d %10.2f %9.1f %12.2f %12.2f %9d" % (n, a[0], a[1] / 1e3, a[1] / a[0], a[2] / 1e3, a[3] / 1e3, a[4]))
    tot_thr = sum(a[2] for a in agg.values()) / span; tot_reg = sum(a[3] for a in agg.values()) / span
    print("time-averaged share of the GPU's thread slots held by running kernels: %.3f ; of its registers: %.3f" % (tot_thr, tot_reg))
    # busy fraction and concurrency histogram via sweep
    ev = []
    for n, s, e, g, b, rg, sm, st in rows:
        ev.append((s, 1)); ev.append((e, -1))
    ev.sort()
    cur, last, hist = 0, t0, collections.Counter()
    for t, dlt in ev:
        hist[cur] += t - last; last = t; cur += dlt
    tot = sum(hist.values())
    print("kernels running concurrently (fraction of time): " + ", ".join("%d:%.2f" % (k, v / tot) for k, v in sorted(hist.items()) if v / tot >= 0.01))
    print("mean concurrency %.1f" % (sum(k * v for k, v in hist.items()) / tot))

if __name__ == "__main__":
    main(sys.argv[1])
