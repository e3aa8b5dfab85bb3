"""ncu launch list (csv, --metrics gpu__time_duration.sum) -> markdown table of ONE train step (between two adam_kernel launches).
usage: python tools/launch_list_md.py <launches.csv> <out.md> "<command line used>" """
import csv, sys
from collections import defaultdict
src, out, cmd = sys.argv[1], sys.argv[2], sys.argv[3]
rows = []
with open(src, newline="") as f:
    rd = csv.reader(l for l in f if l.startswith('"'))
    hdr = next(rd)
    ik, iv, iu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    for r in rd:
        if len(r) <= iv: continue
        v = float(r[iv].replace(",", ""))
        v = v / 1e3 if r[iu] in ("ns", "nsecond") else (v * 1e3 if r[iu] in ("ms", "msecond") else v)      # -> us
        rows.append((r[ik], v))
adam = [i for i, (k, _) in enumerate(rows) if "adam_kernel" in k]
ends = [a for i, a in enumerate(adam) if i + 1 == len(adam) or adam[i + 1] - a > 4]      # last optimizer launch of every step
assert len(ends) >= 2, "need at least two steps to delimit one"
step = rows[ends[-2] + 1: ends[-1] + 1]
agg = defaultdict(lambda: [0, 0.0])
for k, v in step:
    k = k.replace("ga::<unnamed>::", "").replace("void ", "")
    k = k.split("(")[0][:96]
    agg[k][0] += 1; agg[k][1] += v
tot = sum(v for _, v in agg.values())
with open(out, "w") as f:
    f.write("# ncu launch list of ONE stage-1 train step (config 3, B=2 frames)\n\n")
    f.write(f"Command (under gpurun): `{cmd}`\n\nTimes under ncu are cold-cache and serialised: compare SHARES with bench.py's live CUDA-event numbers "
            "(`kernel_ms_per_step`), not absolutes.\n\n")
    f.write(f"Launches in the step: {len(step)}; summed duration {tot / 1e3:.3f} ms\n\n| kernel | launches | total us | share |\n|---|---:|---:|---:|\n")
    for k, (n, v) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        f.write(f"| `{k}` | {n} | {v:.1f} | {100 * v / tot:.1f}% |\n")
print(open(out).read()[:1500])
