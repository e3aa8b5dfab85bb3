"""Summarise an ncu report (raw + source pages) into a small markdown file.
usage: python tools/ncu_summary.py <report.ncu-rep> <out.md> "<title / command>" """
import csv, subprocess, sys
from collections import Counter

rep, out, title = sys.argv[1], sys.argv[2], sys.argv[3]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
idx = {h: i for i, h in enumerate(hdr)}
KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__cycles_active.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
        "smsp__inst_executed.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]
with open(out, "w") as f:
    f.write(f"# {title}\n\nSource: `{rep}` (ncu --set full --clock-control none --import-source on; cold-cache, serialised replays)\n\n")
    for r in rows[2:]:
        f.write(f"## {r[idx['Kernel Name']]}\n\n| metric | value | unit |\n|---|---:|---|\n")
        for k in KEYS:
            if k in idx:
                f.write(f"| `{k}` | {r[idx[k]]} | {units[idx[k]]} |\n")
        f.write("\nWarp stall reasons (per issue-active, `smsp__average_warps_issue_stalled_*`):\n\n")
        st = [(h.split("stalled_")[1].split("_per_")[0], float(r[idx[h]])) for h in hdr if "issue_stalled" in h and "per_issue_active" in h]
        f.write(", ".join(f"{n} {v:.2f}" for n, v in sorted(st, key=lambda t: -t[1]) if v >= 0.05) + "\n\n")
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass"], capture_output=True, text=True).stdout
    srows = list(csv.reader(src.splitlines()))
    his = [i for i, r in enumerate(srows) if r and r[0] == "Address"]
    if his:
        h = srows[his[0]]; si = {x: i for i, x in enumerate(h)}
        end = his[1] - 2 if len(his) > 1 else len(srows)
        data = [r for r in srows[his[0] + 1:end] if len(r) == len(h)]
        tot = sum(int(r[si["Instructions Executed"]]) for r in data) or 1
        c = Counter()
        for r in data:
            t = r[si["Source"]].split()
            if not t:
                continue
            op = (t[1] if t[0].startswith("@") and len(t) > 1 else t[0]).split(".")[0]
            c[op] += int(r[si["Instructions Executed"]])
        f.write("SASS opcode mix of the first kernel (share of executed warp instructions): " +
                ", ".join(f"{op} {100 * n / tot:.1f}%" for op, n in c.most_common(16)) + "\n\n")
        tens = [op for op in c if op.startswith("UTC") or op in ("LDTM", "STTM", "UBLKCP", "UTMALDG", "UTMASTG")]
        f.write("Blackwell-native opcodes present: " + (", ".join(f"{op} x{c[op]}" for op in tens) or "none") + "\n")
print(open(out).read()[:1800])
