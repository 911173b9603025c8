"""Summarise ncu outputs as markdown tables:
   python tools/summarize_ncu.py launches <ncu --csv launch list> <out.md> [n_steps]
   python tools/summarize_ncu.py report   <report.ncu-rep> <out.md>
"""
import collections
import csv
import re
import subprocess
import sys


def launches(src, dst, n_steps=2, cmd=None):
    lines = [l for l in open(src) if not l.startswith("==")]
    agg = collections.OrderedDict()
    for row in csv.DictReader(lines):
        v = float(row["Metric Value"].replace(",", ""))
        u = row["Metric Unit"]
        v = v / 1e3 if u == "ns" else v * 1e3 if u == "ms" else v * 1e6 if u == "s" else v
        key = (re.sub(r"\(.*", "", row["Kernel Name"]).replace("void ", "")[:48], row.get("Grid Size", ""))
        a = agg.setdefault(key, [0, 0.0]); a[0] += 1; a[1] += v
    tot = sum(v[1] for v in agg.values())
    with open(dst, "w") as f:
        f.write(f"# ncu launch list — decode steps of BASELINE configs[1] (Llama-3-8B, B=128, ctx~1664), {n_steps} steps\n\n")
        f.write("`" + (cmd or "OA_CUDA_PROFILER=1 ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none python tools/profile_step.py --steps 2") + "`\n\n")
        f.write(f"Per-launch times are cold-cache and serialised (compare SHARES).  Sum = {tot / n_steps / 1e3:.3f} ms per step.\n\n")
        f.write("| kernel | grid | launches/step | avg us | share |\n|---|---|---:|---:|---:|\n")
        for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| `{k[0]}` | {k[1]} | {v[0] / n_steps:.0f} | {v[1] / v[0]:.1f} | {v[1] / tot * 100:.1f}% |\n")
    print(open(dst).read())


WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers",
        "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct", "smsp__warp_issue_stalled_barrier_per_warp_active.pct"]


def report(src, dst):
    raw = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    with open(dst, "w") as f:
        f.write(f"# ncu --set full captures ({src.split('/')[-1]}; decode step of BASELINE configs[1])\n\n")
        for r in rows[2:]:
            name = re.sub(r"\(.*", "", r[idx["Kernel Name"]]).replace("void ", "")
            f.write(f"## `{name}`  grid {r[idx['Grid Size']]} block {r[idx['Block Size']]}\n\n| metric | value | unit |\n|---|---:|---|\n")
            for w in WANT:
                if w in idx:
                    f.write(f"| {w} | {r[idx[w]]} | {units[idx[w]]} |\n")
            f.write("\n")
    print(open(dst).read()[:3000])


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3], int(sys.argv[4]) if len(sys.argv) > 4 else 2, sys.argv[5] if len(sys.argv) > 5 else None)
    else:
        report(sys.argv[2], sys.argv[3])
