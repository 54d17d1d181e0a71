#!/usr/bin/env python
"""Turn the scratch ncu outputs under gpurun_out/ into the committed summaries under profiles/.
  python tools/ncu_summaries.py launches gpurun_out/launches_r1.csv profiles/launches_r1_summary.md "<command>"
  python tools/ncu_summaries.py raw /tmp/raw.csv   (ncu -i x.ncu-rep --page raw --csv > /tmp/raw.csv) -> metric table on stdout
  python tools/ncu_summaries.py round2 c3 c4       gpurun_out/prof_<wl>_r2_raw.csv (tools/ncu_capture.sh) -> profiles/ncu_<wl>_r2_summary.md
                                                   and profiles/ncu_dram_r2.json (measured DRAM bytes per launch, read by bench.py)
"""
import json
import os
import collections
import csv
import re
import sys

METRICS = [
    "gpu__time_duration.sum", "launch__registers_per_thread", "launch__block_size", "launch__grid_size",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "smsp__thread_inst_executed_per_inst_executed.ratio", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "dram__bytes_read.sum",
    "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__warps_eligible.avg.per_cycle_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
]


def launches(src, dst, command):
    rows = [r for r in csv.reader(l for l in open(src) if l.startswith('"'))]
    hdr, rows = rows[0], rows[1:]
    kn, mv = hdr.index("Kernel Name"), hdr.index("Metric Value")
    agg = collections.OrderedDict()
    for r in rows:
        name = r[kn].split("(")[0].replace("void ", "")
        n, t = agg.get(name, (0, 0.0))
        agg[name] = (n + 1, t + float(r[mv]) / 1e6)
    total = sum(t for _, t in agg.values())
    with open(dst, "w") as f:
        f.write("# ncu launch list (gpu__time_duration.sum, --clock-control none), `%s`\n\n" % command)
        f.write("Raw list: `profiles/%s` (warm-up step + timed step). Serialised, cold-cache times: shares, not absolutes.\n\n" % src.split("/")[-1])
        f.write("| kernel | launches | total ms | share |\n|---|---|---|---|\n")
        for name, (n, t) in agg.items():
            f.write("| `%s` | %d | %.3f | %.1f %% |\n" % (name, n, t, 100 * t / total))


def raw(src):
    rows = list(csv.reader(open(src)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    for m in METRICS:
        if m in hdr:
            i = hdr.index(m)
            print("| `%s` | %s |" % (m, " | ".join((d[i] + " " + units[i]).strip() for d in data)))


def kernel_class(name):
    if "k_nee" in name:
        return "nee"
    if "k_shadow" in name:
        return "shadow"
    if "k_extend" in name:
        return "extend"
    if "k_shade" in name:
        lane = "(bool)1" in name or re.search(r"k_shade<[^>]*,\s*(1|true)>", name)   # k_shade<MODE, LIST>: the handful of deferred rays, side stream
        return "shade_deferred_lane" if lane else "shade"
    return "other"


def round2(workloads):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    dram_path = os.path.join(root, "profiles", "ncu_dram_r2.json")
    try:
        dram = json.load(open(dram_path))
    except Exception:
        dram = {}
    extra = ["smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
             "l1tex__data_pipe_lsu_wavefronts.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum"]
    for wl in workloads:
        src = os.path.join(root, "gpurun_out", "prof_%s_r2_raw.csv" % wl)
        rows = list(csv.reader(open(src)))
        hdr, units, data = rows[0], rows[1], rows[2:]
        kn = hdr.index("Kernel Name")
        names = [d[kn].split("(")[0].replace("void ", "") for d in data]
        agg = {}
        for d, nm in zip(data, names):
            c = agg.setdefault(kernel_class(nm), {"launches": 0, "dram_bytes": 0.0, "ms": 0.0})
            rd, wr = float(d[hdr.index("dram__bytes_read.sum")]), float(d[hdr.index("dram__bytes_write.sum")])
            scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}
            c["dram_bytes"] += rd * scale[units[hdr.index("dram__bytes_read.sum")]] + wr * scale[units[hdr.index("dram__bytes_write.sum")]]
            c["ms"] += float(d[hdr.index("gpu__time_duration.sum")]) * {"ms": 1.0, "us": 1e-3, "s": 1e3}.get(units[hdr.index("gpu__time_duration.sum")], 1.0)
            c["launches"] += 1
        dram[wl] = {k: {"launches": v["launches"], "dram_bytes_per_launch": v["dram_bytes"] / v["launches"], "ms_under_ncu": v["ms"]} for k, v in agg.items()}
        dst = os.path.join(root, "profiles", "ncu_%s_r2_summary.md" % wl)
        with open(dst, "w") as f:
            f.write("# ncu --set full, one timed step of `python bench.py --workload %s --steps 1 --warmup 1 --no-e2e --no-cpu-baseline --no-parity --extra-workloads ''`\n\n" % wl)
            f.write("Capture: `tools/ncu_capture.sh %s` (`prof_%s_r2.ncu-rep`, not kept); this table is `tools/ncu_summaries.py round2 %s`.\n" % (wl, wl, wl))
            f.write("Times under ncu are serialised and cold: compare shares, not absolutes.  Columns = launches in stream order.\n\n")
            f.write("| metric | " + " | ".join("`%s`" % n.replace("k_", "").replace("<(bool)0>", "")[:22] for n in names) + " |\n")
            f.write("|---|" + "---|" * len(names) + "\n")
            for m in METRICS + extra:
                if m in hdr:
                    i = hdr.index(m)
                    cells = []
                    for d in data:
                        try:
                            cells.append("%.4g %s" % (float(d[i]), units[i].replace("register/thread", "").replace("inst", "").strip()))
                        except ValueError:
                            cells.append(d[i])
                    f.write("| `%s` | %s |\n" % (m, " | ".join(c.strip() for c in cells)))
            f.write("\nDRAM bytes per launch (read + write), by kernel class: " + ", ".join("%s %.0f MB x %d" % (k, v["dram_bytes_per_launch"] / 1e6, v["launches"]) for k, v in dram[wl].items()) + ".\n")
        print("wrote", dst)
    json.dump(dram, open(dram_path, "w"), indent=1, sort_keys=True)
    print("wrote", dram_path)


if __name__ == "__main__":
    if sys.argv[1] == "round2":
        round2(sys.argv[2:])
    elif sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3], sys.argv[4])
    else:
        raw(sys.argv[2])
