#!/usr/bin/env python3
"""Summarise an ncu report: per-kernel duration, DRAM bytes, pipe utilisation, stall reasons -> markdown + traffic json.
usage: tools/ncu_traffic.py gpu_out/prof.ncu-rep N_RECORDS gpu_out/ncu_summary.md gpu_out/traffic.json"""
import csv, json, subprocess, sys
rep, nrec, md, js = sys.argv[1], int(sys.argv[2]), sys.argv[3], sys.argv[4]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_elapsed", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio"]
ki = hdr.index("Kernel Name")
out = ["# ncu --set full summary (%s, %d records per launch)\n" % (rep, nrec), "| metric | " + " | ".join(r[ki].split("(")[0][-28:] for r in rows[2:]) + " |", "|---|" + "---|" * (len(rows) - 2)]
traffic = {}
for w in want:
    if w not in hdr:
        continue
    i = hdr.index(w)
    out.append("| %s [%s] | " % (w, units[i]) + " | ".join(r[i] for r in rows[2:]) + " |")
def to_bytes(v, u):
    return float(v) * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
for r in rows[2:]:
    name = r[ki]
    rd, wr = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
    b = to_bytes(r[rd], units[rd]) + to_bytes(r[wr], units[wr])
    key = "k_verify_main" if "k_verify_main<(bool)1>" in name or "k_verify_main<1>" in name else name.split("(")[0].replace("void ", "")
    traffic[key + "_bytes_per_record"] = b / nrec
    for short, metric in (("fmaheavy_pipe_pct", "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed"),
                          ("alu_pipe_pct", "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_elapsed"), ("duration", "gpu__time_duration.sum")):
        if metric in hdr:
            traffic[key + "_" + short] = float(r[hdr.index(metric)].replace(",", ""))
traffic["records_per_launch"] = nrec
open(md, "w").write("\n".join(out) + "\n")
json.dump(traffic, open(js, "w"), indent=1)
print(json.dumps(traffic))
