"""Condense an `ncu --metrics gpu__time_duration.sum,... --csv` launch list into a per-step kernel table
(development aid; the raw list stays next to the summary)."""
import csv
import sys


def load(path):
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    rows = list(csv.reader(lines))
    h = rows[0]
    idx = {n: i for i, n in enumerate(h)}
    recs = {}
    for row in rows[1:]:
        if len(row) < len(h):
            continue
        i = int(row[idx["ID"]])
        rec = recs.setdefault(i, {"name": row[idx["Kernel Name"]], "grid": row[idx["Grid Size"]]})
        rec[row[idx["Metric Name"]]] = float(row[idx["Metric Value"]].replace(",", ""))
    return [recs[i] for i in sorted(recs)]


def main():
    path, first = sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else "conv_first_tc"
    recs = load(path)
    starts = [i for i, r in enumerate(recs) if first in r["name"]]
    if len(starts) < 2:
        print("need two step starts in the capture")
        return
    step = recs[starts[-2]:starts[-1]]           # the last complete step
    total = sum(r["gpu__time_duration.sum"] for r in step) / 1000.0
    print(f"# {path}: last complete step = {len(step)} kernels, sum of durations {total:.1f} us "
          f"(ncu per-launch times are serialised and cold-cache: compare shares, not absolutes)")
    agg = {}
    for r in step:
        nm = r["name"].split("(")[0].replace("void ", "").replace("osvos::", "")
        a = agg.setdefault(nm, [0, 0.0, 0.0, 0.0])
        t = r["gpu__time_duration.sum"] / 1000.0
        a[0] += 1
        a[1] += t
        a[2] += t * r.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0.0)
        a[3] += (r.get("dram__bytes_read.sum", 0.0) + r.get("dram__bytes_write.sum", 0.0)) / 1e6
    print(f"{'kernel':46s} {'n':>3s} {'us':>9s} {'share':>7s} {'tensor-active (time-weighted)':>30s} {'dram MB':>9s}")
    for nm, (c, t, tw, mb) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{nm[:46]:46s} {c:3d} {t:9.1f} {100 * t / total:6.1f}% {tw / t if t else 0:29.1f}% {mb:9.1f}")
    print("\n# launch order")
    for r in step:
        nm = r["name"].split("(")[0].replace("void ", "").replace("osvos::", "")
        mb = (r.get("dram__bytes_read.sum", 0.0) + r.get("dram__bytes_write.sum", 0.0)) / 1e6
        print(f"{nm[:46]:46s} grid {r['grid']:>14s} {r['gpu__time_duration.sum'] / 1000:8.1f} us  tensor "
              f"{r.get('sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 0):5.1f}%  dram {mb:7.1f} MB")


if __name__ == "__main__":
    main()
