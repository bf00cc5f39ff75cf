"""Turn the scratch outputs of scripts/gpu_round.sh <tag> (gpurun_out/) into the tracked summaries under
profiles/: <tag>_launches.md (ncu launch list, per-kernel share), <tag>_ncu_summary.md (key metrics of the
--set full captures) and traffic.json (dram read+write bytes per launch, read back by bench.py).
Usage: python scripts/summarize_profiles.py r1f"""
import collections
import csv
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "gpurun_out")
PROF = os.path.join(ROOT, "profiles")

METRICS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
    "launch__block_size", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "smsp__inst_executed.sum",
    "sm__cycles_active.avg", "sm__cycles_elapsed.avg",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
]
TO_BYTES = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}


def launches(tag):
    path = os.path.join(OUT, f"launches_{tag}.csv")
    lines = [l for l in open(path) if l.startswith('"')]
    rows = list(csv.reader(io.StringIO("".join(lines))))
    hdr, rows = rows[0], rows[1:]
    ik, iv, iu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    tot, cnt = collections.Counter(), collections.Counter()
    for r in rows:
        scale = {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(r[iu], 1e-3)
        v = float(r[iv].replace(",", "")) * scale
        k = r[ik].split("(")[0]
        tot[k] += v
        cnt[k] += 1
    total = sum(tot.values())
    out = [f"# {tag} — ncu launch list of `python bench.py --steps 5 --warmup 3 --no-cpu` (all workloads)", "",
           "`ncu --metrics gpu__time_duration.sum --clock-control none -c 1200` (cold-cache, serialised: compare "
           "shares, not absolutes).", f"Raw CSV: gpurun_out/launches_{tag}.csv (first 1200 launches).", "",
           "| kernel | launches | total us | share | avg us |", "|---|---|---|---|---|"]
    for k, v in tot.most_common():
        out.append(f"| `{k}` | {cnt[k]} | {v:.1f} | {100 * v / total:.1f} % | {v / cnt[k]:.2f} |")
    open(os.path.join(PROF, f"{tag}_launches.md"), "w").write("\n".join(out) + "\n")


def captures(tag):
    out = [f"# {tag} — ncu summary of the three hot kernels (H100, `--set full --clock-control none`)", "",
           f"Captured by `scripts/gpu_round.sh {tag}` (`ncu ... -k regex:<kernel> -s 2 -c 2 python bench.py --steps 4 "
           "--warmup 3 --no-cpu --workload <w>`);", f"raw reports `gpurun_out/prof_{{ekf,pf,mpc}}_{tag}.ncu-rep` "
           "(scratch, not tracked).  Durations under ncu are cold-cache and serialised; bench numbers are CUDA-event "
           "timed.", "`traffic` = dram read + write per launch (what `profiles/traffic.json` holds; write-backs still "
           "sitting in the 126 MB L2 when the kernel ends are not in it, which is why EKF/PF writes look small).", ""]
    traffic = {}
    for w in ("ekf", "pf", "mpc"):
        rep = os.path.join(OUT, f"prof_{w}_{tag}.ncu-rep")
        if not os.path.exists(rep):
            continue
        txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(io.StringIO(txt)))
        hdr, units, data = rows[0], rows[1], rows[2:]
        name = data[0][hdr.index("Kernel Name")].split("(")[0]
        out += [f"## {w}: `{name}`", "", "| metric | " + " | ".join(f"launch {i + 1}" for i in range(len(data))) + " |",
                "|---|" + "---|" * len(data)]
        for m in METRICS:
            if m in hdr:
                i = hdr.index(m)
                out.append(f"| {m} | " + " | ".join(f"{d[i]} {units[i]}" for d in data) + " |")
        ir, iw = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
        t = [float(d[ir].replace(",", "")) * TO_BYTES[units[ir]] + float(d[iw].replace(",", "")) * TO_BYTES[units[iw]]
             for d in data]
        sys.path.insert(0, ROOT)
        import bench
        traffic[w] = {"bytes": sum(t) / len(t), "stamp": bench.kernel_stamp(w), "kernel": name, "capture": tag}
        out.append("")
    open(os.path.join(PROF, f"{tag}_ncu_summary.md"), "w").write("\n".join(out))
    path = os.path.join(PROF, "traffic.json")
    try:
        merged = json.load(open(path))
    except Exception:
        merged = {}
    merged.update(traffic)
    json.dump(merged, open(path, "w"), indent=1)
    return traffic


if __name__ == "__main__":
    tag = sys.argv[1] if len(sys.argv) > 1 else "r1"
    launches(tag)
    print(captures(tag))
