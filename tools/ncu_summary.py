"""Turn ncu outputs into markdown summaries.

    python tools/ncu_summary.py launches launches.csv launches.md "title"
    python tools/ncu_summary.py full prof.ncu-rep kernels.md [traffic.json]

`launches`: per-kernel share of the step from `ncu --metrics gpu__time_duration.sum` (cold-cache,
serialised: compare SHARES, not absolutes). `full`: key metrics of each captured kernel from
`ncu --set full` (read here with `ncu -i ... --page raw --csv`).
"""
import collections
import csv
import io
import json
import re
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("launch__registers_per_thread", "registers/thread"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active %"),
    ("l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "L1/TEX throughput %"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 throughput %"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput %"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate %"),
    ("l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum", "global load requests"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "global load sectors"),
    ("l1tex__t_requests_pipe_lsu_mem_global_op_red.sum", "global RED requests"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_red.sum", "global RED sectors"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_scoreboard / issue"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait / issue"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short_scoreboard / issue"),
    ("smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "stall lg_throttle / issue"),
    ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "stall mio_throttle / issue"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier / issue"),
    ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall math_pipe / issue"),
]


def short(name):
    return re.sub(r"\(.*", "", name).replace("void ", "")[:70]


def launches(src, dst, title):
    lines = [l for l in open(src) if not l.startswith("==")]
    agg = collections.OrderedDict()
    for row in csv.DictReader(lines):
        if row.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(row["Metric Value"].replace(",", ""))
        v = {"ns": v / 1e3, "us": v, "ms": v * 1e3, "s": v * 1e6}.get(row["Metric Unit"], v)
        a = agg.setdefault(short(row["Kernel Name"]), [0, 0.0])
        a[0] += 1
        a[1] += v
    tot = sum(a[1] for a in agg.values())
    out = ["# " + title, "", "Source: `%s` (`ncu --metrics gpu__time_duration.sum --clock-control none`)." % src,
           "Per-launch times under ncu are cold-cache and serialised: read the SHARE column.", "",
           "| share | launches | avg us | kernel |", "|---:|---:|---:|---|"]
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        out.append("| %.1f%% | %d | %.1f | `%s` |" % (100 * t / tot, n, t / n, k))
    out.append("")
    out.append("total %.1f us over %d launches" % (tot, sum(a[0] for a in agg.values())))
    open(dst, "w").write("\n".join(out) + "\n")
    print("\n".join(out))


def full(src, dst, traffic_json=None):
    raw = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                         text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    kn = idx["Kernel Name"]
    by_kernel = collections.OrderedDict()
    for r in rows[2:]:
        by_kernel.setdefault(short(r[kn]), []).append(r)
    out = ["# ncu --set full: key metrics per kernel", "", "Source: `%s`, read with `ncu -i ... --page raw --csv`." % src,
           "Values are the mean over the captured launches of each kernel.", ""]
    traffic = {}
    for k, rs in by_kernel.items():
        out += ["## `%s`  (%d launches captured)" % (k, len(rs)), "", "| metric | value |", "|---|---:|"]
        for key, label in KEYS:
            if key not in idx:
                continue
            vals = []
            for r in rs:
                try:
                    vals.append(float(r[idx[key]].replace(",", "")))
                except ValueError:
                    pass
            if not vals:
                continue
            v = sum(vals) / len(vals)
            out.append("| %s (`%s`) | %.4g %s |" % (label, key, v, units[idx[key]]))
        def mean_bytes(key):
            u = units[idx[key]]
            mul = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
            vs = [float(r[idx[key]].replace(",", "")) * mul for r in rs]
            return sum(vs) / len(vs)
        if "dram__bytes_read.sum" in idx:
            t = mean_bytes("dram__bytes_read.sum") + mean_bytes("dram__bytes_write.sum")
            traffic[k.split("<")[0] + "_dram_bytes_per_launch"] = t
            out.append("| **DRAM traffic per launch (read+write)** | %.4g MB |" % (t / 1e6))
        out.append("")
    open(dst, "w").write("\n".join(out) + "\n")
    if traffic_json:
        merged = {}
        try:
            merged = json.load(open(traffic_json))  # one capture per kernel: keep the other kernels' entries
        except Exception:
            pass
        merged.update(traffic)
        json.dump(merged, open(traffic_json, "w"), indent=1)
    print("\n".join(out))


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3], sys.argv[4] if len(sys.argv) > 4 else "kernel launch list")
    else:
        full(sys.argv[2], sys.argv[3], sys.argv[4] if len(sys.argv) > 4 else None)
