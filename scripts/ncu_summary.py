#!/usr/bin/env python
"""Turn an ncu launch list (csv) + one `--set full` report into the markdown / json kept under profiles/.

    python scripts/ncu_summary.py --launches gpurun_out/launches.csv --report gpurun_out/prof_r01.ncu-rep \
        --title "Round 1 ..." --out profiles/r01_ncu_summary.md [--traffic profiles/dram_traffic.json]

Reads the report with `ncu -i ... --page raw --csv` (works without a GPU).
"""
import argparse
import csv
import io
import json
import subprocess
from collections import OrderedDict

METRICS = [
    "gpu__time_duration.sum",
    "dram__bytes_read.sum",
    "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread",
    "launch__waves_per_multiprocessor",
    "smsp__inst_executed.sum",
    "smsp__thread_inst_executed_per_inst_executed.ratio",
    "l1tex__t_sector_hit_rate.pct",
    "lts__t_sector_hit_rate.pct",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
]


def short(name):
    name = name.split("(")[0]
    return name.replace("delora::", "").replace("void ", "")


def read_launches(path):
    rows = []
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    for r in csv.DictReader(io.StringIO("".join(lines))):
        if r.get("Metric Name") == "gpu__time_duration.sum":
            v = float(r["Metric Value"].replace(",", ""))
            unit = r.get("Metric Unit", "ns")
            scale = {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(unit, 1e-3)
            rows.append((short(r["Kernel Name"]), v * scale))
    agg = OrderedDict()
    for k, us in rows:
        agg.setdefault(k, []).append(us)
    return agg


def read_report(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rd = list(csv.reader(io.StringIO(out)))
    header, units = rd[0], rd[1]
    res = OrderedDict()
    for row in rd[2:]:
        d = dict(zip(header, row))
        k = short(d["Kernel Name"])
        if k in res:
            continue
        res[k] = {m: (d.get(m, ""), units[header.index(m)] if m in header else "") for m in METRICS}
    return res


def to_bytes(val, unit):
    v = float(val.replace(",", ""))
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches")
    ap.add_argument("--report")
    ap.add_argument("--title", default="ncu summary")
    ap.add_argument("--out", required=True)
    ap.add_argument("--traffic")
    a = ap.parse_args()
    md = [f"# {a.title}", ""]
    if a.launches:
        agg = read_launches(a.launches)
        per_launch_total = sum(sum(v) for v in agg.values())
        md += ["## Launch list", "", "| kernel | launches | mean µs | share of captured time |", "|---|---|---|---|"]
        for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
            md.append(f"| `{k}` | {len(v)} | {sum(v) / len(v):.1f} | {100 * sum(v) / per_launch_total:.1f} % |")
        md.append("")
    if a.report:
        rep = read_report(a.report)
        md += ["## Per-kernel metrics (ncu --set full, one launch each)", ""]
        traffic = {}
        for k, ms in rep.items():
            md += [f"### `{k}`", "", "| metric | value |", "|---|---|"]
            for m in METRICS:
                val, unit = ms[m]
                if val != "":
                    md.append(f"| {m} | {val} {unit} |")
            md.append("")
            try:
                traffic[k] = {
                    "dram_bytes_read": to_bytes(*ms["dram__bytes_read.sum"]),
                    "dram_bytes_write": to_bytes(*ms["dram__bytes_write.sum"]),
                    "warp_instructions": float(ms["smsp__inst_executed.sum"][0].replace(",", "")),
                }
                traffic[k]["dram_bytes"] = traffic[k]["dram_bytes_read"] + traffic[k]["dram_bytes_write"]
            except Exception:
                pass
        if a.traffic:
            # bench.py reads the per-OPERATOR totals (operator = the kernels one C-ABI call launches)
            ops = {"projection": ("project_scatter_kernel", "project_resolve_kernel"),
                   "normals": ("normals_7x11_kernel",),
                   "icp": ("icp_dense_kernel", "icp_dense_pending_kernel", "icp_finalize_kernel", "target_extents_kernel")}
            doc = {}
            for op, names in ops.items():
                tot = sum(t["dram_bytes"] for k, t in traffic.items() if k.split("<")[0] in names)
                if tot:
                    doc[op] = tot
            doc["_source"] = (f"{a.out}: dram__bytes_read.sum + dram__bytes_write.sum per launch "
                              "(ncu --set full, one launch per kernel)")
            doc["_per_kernel"] = {k: t["dram_bytes"] for k, t in traffic.items()}
            # warp instructions per launch of every operator (issue-slot utilisation = this / (time x SMs x 4 x clock))
            doc["_warp_instructions"] = {op: sum(t["warp_instructions"] for k, t in traffic.items() if k.split("<")[0] in names)
                                         for op, names in ops.items()}
            with open(a.traffic, "w") as f:
                json.dump(doc, f, indent=1)
    with open(a.out, "w") as f:
        f.write("\n".join(md) + "\n")
    print("wrote", a.out)


if __name__ == "__main__":
    main()
