"""Turns Nsight Compute outputs (CSV launch lists, .ncu-rep reports) into small text summaries for profiles/.

    python tools/summarize_ncu.py launches launches_step.csv > profiles/launches_step.md
    python tools/summarize_ncu.py report pcg.ncu-rep > profiles/pcg_kernels.md
"""
import collections
import csv
import io
import re
import subprocess
import sys

METRICS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_bytes.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
    "launch__grid_size", "launch__block_size", "inst_executed", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "launch__occupancy_limit_registers", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
]


def short(name):
    name = re.sub(r"\(.*", "", name)
    return name.replace("blub::<unnamed>::", "").replace("void ", "").replace("unnamed>::", "")


def launches(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    agg = collections.OrderedDict()
    tot = 0.0
    for row in csv.DictReader(lines):
        if row.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(row["Metric Value"].replace(",", ""))
        v = {"ns": v / 1e3, "us": v, "ms": v * 1e3}.get(row["Metric Unit"], v)
        k = short(row["Kernel Name"])
        a = agg.setdefault(k, [0, 0.0])
        a[0] += 1
        a[1] += v
        tot += v
    print(f"# ncu launch list: {path}\n\n`ncu --metrics gpu__time_duration.sum --clock-control none` (cold-cache, serialised: compare SHARES)\n")
    print(f"total {tot:.1f} us over {sum(a[0] for a in agg.values())} launches\n")
    print("| kernel | launches | total us | avg us | share |\n|---|---:|---:|---:|---:|")
    for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"| `{k}` | {c} | {t:.1f} | {t / c:.1f} | {100 * t / tot:.1f}% |")


def report(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    print(f"# ncu --set full: {path}\n")
    for r in rows[2:]:
        print(f"## `{short(r[idx['Kernel Name']])}`  grid {r[idx['launch__grid_size']]} x block {r[idx['launch__block_size']]}\n")
        print("| metric | value | unit |\n|---|---:|---|")
        for m in METRICS:
            if m in idx:
                print(f"| {m} | {r[idx[m]]} | {units[idx[m]]} |")
        stalls = []
        for h, i in idx.items():
            if "issue_stalled" in h and "per_issue_active" in h and r[i] not in ("0", "n/a", ""):
                stalls.append((h.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", ""), float(r[i].replace(",", ""))))
        stalls.sort(key=lambda kv: -kv[1])
        print("\nwarp stall reasons (warps per issue-active cycle): " + ", ".join(f"{a} {b:.2f}" for a, b in stalls[:7]))
        print()


def traffic(path):
    """dram bytes of the persistent PCG solve kernel, as JSON."""
    import json

    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
    best = None
    for r in rows[2:]:
        if "pcg_solve_persistent" not in r[idx["Kernel Name"]]:
            continue
        rd = float(r[idx["dram__bytes_read.sum"]]) * scale[units[idx["dram__bytes_read.sum"]]]
        wr = float(r[idx["dram__bytes_write.sum"]]) * scale[units[idx["dram__bytes_write.sum"]]]
        t = r[idx["gpu__time_duration.sum"]] + " " + units[idx["gpu__time_duration.sum"]]
        best = {"dram_bytes_per_solve": int(rd + wr), "dram_read": int(rd), "dram_write": int(wr), "kernel_time_under_ncu": t,
                "kernel": "pcg_solve_persistent_kernel (256^3 all-fluid microbench, 33 iterations)", "source": path}
    print(json.dumps(best, indent=1))


if __name__ == "__main__":
    {"launches": launches, "report": report, "traffic": traffic}[sys.argv[1]](sys.argv[2])
