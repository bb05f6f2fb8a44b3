"""Summarise an `ncu --set full` report (read here, no GPU needed) into a JSON file: key raw metrics and the
per-opcode dynamic instruction census from the source page.
    python tools/summarize_ncu.py profile_out/r2_prof_merkle4.ncu-rep merkle4_2p20 profile_out/ncu_summary.json"""
import collections
import csv
import io
import json
import re
import subprocess
import sys

KEYS = {
    "gpu__time_duration.sum": "duration_ms",
    "dram__bytes_read.sum": "dram_read_MB",
    "dram__bytes_write.sum": "dram_write_MB",
    "launch__registers_per_thread": "registers_per_thread",
    "sm__warps_active.avg.per_cycle_active": "warps_active_per_sm",
    "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed": "pipe_fmaheavy_active_pct",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active": "inst_pipe_fma_pct",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active": "inst_pipe_alu_pct",
    "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active": "inst_pipe_fp64_pct",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active": "inst_pipe_xu_pct",
    "smsp__issue_active.avg.pct_of_peak_sustained_active": "issue_active_pct",
    "smsp__inst_executed.sum": "warp_instructions",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed": "sm_throughput_pct",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed": "dram_throughput_pct",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum": "global_ld_sectors",
    "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum": "global_ld_requests",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum": "global_st_sectors",
    "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum": "global_st_requests",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum": "smem_bank_conflicts",
    "sm__cycles_elapsed.avg.per_second": "sm_clock_ghz",
}
STALLS = "smsp__average_warps_issue_stalled_"


def page(rep, name):
    out = subprocess.run(["ncu", "-i", rep, "--page", name, "--csv"], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main():
    rep, label, dst = sys.argv[1], sys.argv[2], sys.argv[3]
    rows = page(rep, "raw")
    hdr, units, vals = rows[0], rows[1], rows[2]
    res = {"kernel": vals[hdr.index("Kernel Name")].split("(")[0], "grid": vals[hdr.index("Grid Size")],
           "block": vals[hdr.index("Block Size")], "stalls_per_issue": {}}
    scale = {"Gbyte": 1e3, "Mbyte": 1.0, "Kbyte": 1e-3, "byte": 1e-6, "s": 1e3, "ms": 1.0, "us": 1e-3, "ns": 1e-6}
    for h, u, v in zip(hdr, units, vals):
        if h in KEYS:
            try:
                f = float(v)
                if KEYS[h].endswith("_MB") or KEYS[h].endswith("_ms"):
                    f *= scale.get(u, 1.0)          # ncu picks the unit per value; normalise to MB / ms
                res[KEYS[h]] = f
            except ValueError:
                res[KEYS[h]] = v
        elif h.startswith(STALLS) and h.endswith("_per_issue_active.ratio"):
            try:
                f = float(v)
            except ValueError:
                continue
            if f >= 0.05:
                res["stalls_per_issue"][h[len(STALLS):-len("_per_issue_active.ratio")]] = round(f, 3)
    res["dram_bytes_per_launch"] = int((res.get("dram_read_MB", 0) + res.get("dram_write_MB", 0)) * 1e6)
    if res.get("global_ld_requests"):
        res["global_ld_sectors_per_request"] = res["global_ld_sectors"] / res["global_ld_requests"]
        res["global_st_sectors_per_request"] = res["global_st_sectors"] / res["global_st_requests"]
    # per-opcode census from the source page
    rows = page(rep, "source")
    hdr = rows[1]
    i_s, i_e = hdr.index("Source"), hdr.index("Instructions Executed")
    ops = collections.Counter()
    static = 0
    for r in rows[2:]:
        if len(r) <= i_e:
            continue
        m = re.match(r"(@!?U?P\d+\s+)?([A-Z0-9_.]+)", r[i_s].strip())
        if not m:
            continue
        static += 1
        op = m.group(2)
        key = op.split(".")[0]
        if key == "IMAD":
            key = "IMAD.WIDE" if "WIDE" in op else ("IMAD.HI" if "HI" in op else ("IMAD.MOV" if "MOV" in op else "IMAD.other"))
        ops[key] += int(r[i_e])
    warps = res.get("warp_instructions", 0) and int(vals[hdr.index("Source")] if False else 0)
    grid = int(re.findall(r"\d+", res["grid"])[0])
    block = int(re.findall(r"\d+", res["block"])[0])
    nwarps = grid * block // 32
    res["static_sass_instructions"] = static
    res["warp_instructions_per_warp"] = {k: round(v / nwarps, 1) for k, v in ops.most_common(16)}
    res["warp_instructions_per_warp"]["TOTAL"] = round(sum(ops.values()) / nwarps, 1)
    try:
        with open(dst) as f:
            allres = json.load(f)
    except Exception:
        allres = {}
    allres[label] = res
    with open(dst, "w") as f:
        json.dump(allres, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
