"""Per-warp phase timeline of one iteration of the persistent EM kernel (dev helper).
usage: timeline_em.py [C] [key=value ...]      (sb_em_set_option keys, e.g. rebalance=0)"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from salmon_b200 import EMContext, default_params
from salmon_b200.synth import synth_eq
C = int(sys.argv[1]) if len(sys.argv) > 1 else 500000
eq, proj, eff, uniq = synth_eq(seed=1, C=C, M=C // 2, total_count=40 * C)
ctx = EMContext(0)
for kv in sys.argv[2:]:
    k, v = kv.split("=")
    ctx.set_option(k, int(v))
p = default_params(min_iter=60, max_iter=60)
ctx.upload(eq, proj, eff, uniq); ctx.prepare(p)
ctx.run()
nw = ctx.arm_timeline(40)
r = ctx.run()
t = ctx.read_timeline(nw).astype(np.int64)
t0 = t[:, 0].min()
names = ["P1 start", "P1 end", "bar1 end", "P2 start", "P2 end", "reduce end", "bar2 end"]
sizes = (eq.off[1:] - eq.off[:-1]).astype(np.int64)
tc = np.bincount(eq.tids[np.repeat(sizes > 1, sizes)], minlength=eq.n_txps)
print("classes >32:", int((sizes > 32).sum()), " txps >32:", int((tc > 32).sum()), ">256:", int((tc > 256).sum()), ">2048:", int((tc > 2048).sum()), "max", int(tc.max()), " entries in txp rows >32:", int(tc[tc > 32].sum()))
print("C", C, "loop us/iter", r.loop_kernel_ms / 60 * 1e3, "warps", nw)
sb = ctx.info("stream_bytes")
print("stream per iteration: %.2f MB (class-major %.2f, transcript-major %.2f; SELL columns %d / %d; long-row entries %d / %d; "
      "fallback rows %d / %d) = %.0f GB/s" % (
          sb / 1e6, ctx.info("stream_bytes_cm") / 1e6, ctx.info("stream_bytes_tm") / 1e6, ctx.info("sell_cols_cm"),
          ctx.info("sell_cols_tm"), ctx.info("long_entries_cm"), ctx.info("long_entries_tm"), ctx.info("fallback_rows_cm"),
          ctx.info("fallback_rows_tm"), sb / (r.loop_kernel_ms / 60 * 1e-3) / 1e9))
for i, n in enumerate(names):
    col = t[:, i] - t0
    print(f"{n:11s} min {col.min()/1e3:8.2f}  p50 {np.median(col)/1e3:8.2f}  p90 {np.percentile(col,90)/1e3:8.2f}  max {col.max()/1e3:8.2f} us")
d1 = (t[:, 1] - t[:, 0]) / 1e3; d2 = (t[:, 4] - t[:, 3]) / 1e3
print("P1 duration per warp: p50 %.2f p90 %.2f p99 %.2f max %.2f us" % (np.median(d1), np.percentile(d1, 90), np.percentile(d1, 99), d1.max()))
print("P2 duration per warp: p50 %.2f p90 %.2f p99 %.2f max %.2f us" % (np.median(d2), np.percentile(d2, 90), np.percentile(d2, 99), d2.max()))
d3 = (t[:, 7] - t[:, 3]) / 1e3
print("P2 home stream per warp: p50 %.2f p90 %.2f max %.2f us ; queue part p50 %.2f max %.2f" % (np.median(d3), np.percentile(d3, 90), d3.max(), np.median(d2 - d3), (d2 - d3).max()))
# the grid barrier after a phase waits for the last warp: how long after the median warp it ends
for ph, (c_end, c_start) in (("P1", (1, 0)), ("P2", (4, 3))):
    end = (t[:, c_end] - t0) / 1e3
    print("%s end: median warp %.2f us, last warp %.2f us, gap %.2f us" % (ph, np.median(end), end.max(), end.max() - np.median(end)))


def items(row, base):
    lr = int(row[base])
    return "long rows %3d (%6d entries, longest %4d)" % (lr >> 32, lr & 0xFFFFFFFF, int(row[base + 1]))


for ph, (c_start, c_end, c_home, q_base) in (("P1", (0, 1, 8, 9)), ("P2", (3, 4, 7, 11))):
    d = t[:, c_end] - t[:, c_start]
    print("10 slowest %s warps (us from the warp's phase start):" % ph)
    for w in np.argsort(-d)[:10]:
        home = (t[w, c_home] - t[w, c_start]) / 1e3
        print("  warp %5d  home end %7.2f  phase end %7.2f  %s" % (w, home, d[w] / 1e3, items(t[w], q_base)))
