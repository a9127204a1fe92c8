"""Per-resolution kernel-class table from the ncu launch lists of scripts/sweep_ncu.sh (BASELINE.json configs[4]):
time, time-weighted tensor-pipe activity and achieved DRAM GB/s per kernel class (ncu per-launch times are serialised
and cold-cache: read the tensor % and bytes, compare shares)."""
import glob
import sys

from summarize_launches import load

prefix = sys.argv[1]
peaks = {"hbm": 3350.0}   # GB/s, H100 SXM data sheet (HBM3)
for path in sorted(glob.glob(prefix + "*.csv"), key=lambda p: int(p.split("_")[-1].split("x")[0])):
    res = path.split("_")[-1].replace(".csv", "")
    recs = load(path)
    total = sum(r["gpu__time_duration.sum"] for r in recs) / 1000.0
    print(f"\n== {res}: {len(recs)} kernels, sum of durations {total:.1f} us")
    print(f"{'kernel class':28s} {'n':>3s} {'us':>8s} {'share':>7s} {'tensor-active':>14s} {'dram MB':>9s} {'dram GB/s':>10s} {'of HBM peak':>12s}")
    agg = {}
    for r in recs:
        nm = r["name"].split("(")[0].split("<")[0].replace("void ", "").replace("osvos::", "")
        a = agg.setdefault(nm, [0, 0.0, 0.0, 0.0])
        t = r["gpu__time_duration.sum"] / 1000.0
        a[0] += 1
        a[1] += t
        a[2] += t * r.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0.0)
        a[3] += (r.get("dram__bytes_read.sum", 0.0) + r.get("dram__bytes_write.sum", 0.0)) / 1e6
    for nm, (c, t, tw, mb) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        gbs = mb / t * 1e3 if t else 0.0          # MB / us = TB/s -> GB/s
        print(f"{nm[:28]:28s} {c:3d} {t:8.1f} {100 * t / total:6.1f}% {tw / t if t else 0:13.1f}% {mb:9.1f} {gbs:10.0f} {gbs / peaks['hbm']:11.1%}")
