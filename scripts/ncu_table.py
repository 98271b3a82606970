"""Condense an `ncu --page raw --csv` dump (one row per profiled launch; kept instead of the .ncu-rep, which is
>100 MB for ~50 kernels with the full metric set) into the per-kernel table kept under profiles/:
duration, DRAM bytes and achieved GB/s against the measured HBM peak, tensor / MUFU / issue utilisation, launch shape.

    python scripts/ncu_table.py gpurun_out/r02a_ncu_all_raw.csv profiles/r02a_ncu_all_kernels.csv [targets.log]
"""
import csv
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLS = [("gpu__time_duration.sum", "duration_us"), ("dram__bytes_read.sum", "dram_read_MB"), ("dram__bytes_write.sum", "dram_write_MB"),
        ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct_of_peak"),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor_pipe_pct"),
        ("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_elapsed", "mufu_pipe_pct"),
        ("sm__issue_active.avg.pct_of_peak_sustained_elapsed", "issue_pct"),
        ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm_throughput_pct"),
        ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "l2_throughput_pct"),
        ("launch__registers_per_thread", "regs"), ("launch__grid_size", "grid"), ("launch__block_size", "block"),
        ("launch__shared_mem_per_block_dynamic", "dyn_smem_B")]
SCALE = {"ns": 1e-3, "nsecond": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "s": 1e6, "second": 1e6,
         "byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}


def main():
    src, dst = sys.argv[1], sys.argv[2]
    rows = list(csv.reader(open(src)))
    hdr = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    names, units = rows[hdr], rows[hdr + 1]
    peak = 6574.1
    mp = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(mp):
        peak = json.load(open(mp)).get("hbm_gbs", peak)
    targets = []
    if len(sys.argv) > 3 and os.path.exists(sys.argv[3]):
        m = re.search(r"targets: (.*)", open(sys.argv[3]).read())
        targets = m.group(1).strip().split(",") if m else []
    out = []
    for r in rows[hdr + 2:]:
        rec = {"kernel": re.sub(r"\(.*", "", r[names.index("Kernel Name")]).replace("void ", "")[:90]}
        for col, key in COLS:
            if col not in names:
                continue
            i = names.index(col)
            try:
                v = float(r[i].replace(",", ""))
            except ValueError:
                continue
            rec[key] = round(v * SCALE.get(units[i], 1.0), 3)
        if "duration_us" in rec and rec["duration_us"] > 0:
            gbs = (rec.get("dram_read_MB", 0) + rec.get("dram_write_MB", 0)) / rec["duration_us"] * 1e3
            rec["dram_GBps"] = round(gbs, 1)
            rec["dram_frac_of_measured_hbm_peak"] = round(gbs / peak, 3)
        out.append(rec)
    keys = ["kernel"] + [k for _, k in COLS] + ["dram_GBps", "dram_frac_of_measured_hbm_peak"]
    with open(dst, "w", newline="") as fh:
        w = csv.DictWriter(fh, fieldnames=keys)
        w.writeheader()
        for rec in out:
            w.writerow({k: rec.get(k, "") for k in keys})
    print(len(out), "launches ->", dst, "(targets in launch order:", ",".join(targets) + ")")


if __name__ == "__main__":
    main()
