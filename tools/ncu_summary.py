#!/usr/bin/env python
"""Summarise an .ncu-rep (read here, without a GPU): key raw metrics of the first matching
kernel as JSON, and the top stalled SASS instructions of its source page.

    python tools/ncu_summary.py prof.ncu-rep [--top 40] [--json out.json]"""
import argparse
import csv
import io
import json
import subprocess

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_atom.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_ld.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared_op_st.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_tag_requests.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "launch__block_size", "launch__grid_size", "launch__registers_per_thread", "launch__occupancy_limit_shared_mem",
        "launch__occupancy_limit_registers", "sm__cycles_active.avg", "sm__cycles_elapsed.avg",
        "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__warps_eligible.avg.per_cycle_active"]


def raw(rep, match=""):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    kn = hdr.index("Kernel Name")
    first = next((r for r in rows[2:] if match in r[kn]), rows[2])  # first launch whose name contains `match`
    d = {}
    for h, u, v in zip(hdr, units, first):
        if h in KEYS or h.startswith("smsp__average_warps_issue_stalled") and h.endswith("per_issue_active.ratio"):
            d[f"{h} [{u}]" if u else h] = v
        if h == "Kernel Name":
            d["kernel"] = v
    return d


def source(rep, top):
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    start = next(i for i, r in enumerate(rows) if r and r[0] == "Address")
    hdr = rows[start]
    ix = {h: i for i, h in enumerate(hdr)}
    data = []
    for r in rows[start + 1:]:
        if len(r) < len(hdr) or r[0] == "Address" or not r[0].startswith("0x"):
            if r and r[0] == "Kernel Name":
                break
            continue
        data.append(r)
    tot = sum(int(r[ix["# Samples"]]) for r in data)
    print("total samples", tot, "instructions", len(data))
    stalls = [h for h in hdr if h.startswith("stall_") and "Not Issued" not in h]
    agg = {s: sum(int(r[ix[s]]) for r in data) for s in stalls}
    print("stall totals:", {k: v for k, v in sorted(agg.items(), key=lambda kv: -kv[1]) if v})
    for r in sorted(data, key=lambda r: -int(r[ix["# Samples"]]))[:top]:
        st = {k[6:]: int(r[ix[k]]) for k in stalls if int(r[ix[k]]) > 0}
        print(r[ix["# Samples"]].rjust(6), r[ix["Source"]].strip()[:64].ljust(64), r[ix["Instructions Executed"]].rjust(8), st)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("rep")
    ap.add_argument("--top", type=int, default=40)
    ap.add_argument("--json", default="")
    ap.add_argument("--match", default="", help="summarise the first launch whose kernel name contains this")
    ap.add_argument("--no-source", action="store_true")
    a = ap.parse_args()
    d = raw(a.rep, a.match)
    print(json.dumps(d, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(d, f, indent=1)
    if not a.no_source:
        source(a.rep, a.top)
