#!/usr/bin/env python
"""Turn an `ncu --set full` capture into the compact per-launch text that goes under profiles/.

    python tools/ncu_summary.py gpurun_out/prof.ncu-rep [--match REGEX] [--json OUT.json] > profiles/rNN_<what>_ncu.txt

Runs `ncu -i <rep> --page raw --csv` (ncu is installed in the CPU container; no GPU needed to read a report) and keeps the
metrics the roofline discussion uses: duration, DRAM bytes, tensor-pipe / L2 / DRAM utilisation, store efficiency,
registers, instruction count.  With --json it also writes the mean DRAM traffic per launch in the shape bench.py reads from
profiles/gemm_traffic.json (`roofline.traffic`).  A CSV produced earlier can be passed instead of a .ncu-rep.
"""
import argparse
import csv
import io
import json
import re
import subprocess
import sys

KEEP = [
    "gpu__time_duration.sum",
    "dram__bytes_read.sum",
    "dram__bytes_write.sum",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tensor",            # prefix match: the spelling differs between ncu releases
    "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "launch__registers_per_thread",
    "launch__grid_size",
    "launch__cluster_size",
    "smsp__inst_executed.sum",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active",
]


def read_rows(path):
    if path.endswith(".csv"):
        text = open(path).read()
    else:
        text = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], check=True, capture_output=True, text=True).stdout
    lines = [l for l in text.splitlines() if not l.startswith("==")]
    return list(csv.reader(io.StringIO("\n".join(lines))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("report")
    ap.add_argument("--match", default=".", help="regex on the kernel name")
    ap.add_argument("--json", default=None, help="write mean DRAM bytes per launch (bench.py's roofline.traffic source)")
    ap.add_argument("--note", default="", help="first comment line of the summary")
    args = ap.parse_args()
    rows = read_rows(args.report)
    if len(rows) < 3:
        sys.exit("empty report")
    header, units = rows[0], rows[1]
    name_col = header.index("Kernel Name")
    cols = [i for i, h in enumerate(header) if any(h == k or h.startswith(k) for k in KEEP)]
    print(f"# {args.note or 'ncu --set full --clock-control none'}; source {args.report}")
    per = []
    n = 0
    for r in rows[2:]:
        if len(r) <= name_col or not re.search(args.match, r[name_col]):
            continue
        print(f"launch {n}: {r[name_col][:160]}")
        rec = {"kernel": r[name_col][:100]}
        for i in cols:
            val = r[i].replace(",", "")
            print(f"    {header[i]} [{units[i]}] = {val}")
            try:
                rec[header[i] + " [" + units[i] + "]"] = float(val)
            except ValueError:
                pass
        per.append(rec)
        n += 1
    if args.json and per:
        def to_bytes(rec, key):
            for k, v in rec.items():
                if k.startswith(key):
                    unit = k[k.index("[") + 1:-1].lower()
                    mult = {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(unit, 1)
                    return v * mult
            return 0.0
        tot = [to_bytes(p, "dram__bytes_read.sum") + to_bytes(p, "dram__bytes_write.sum") for p in per]
        json.dump({"dram_bytes_per_launch": sum(tot) / len(tot), "source": f"{args.report}: mean over {len(tot)} launches matching /{args.match}/",
                   "per_launch": per}, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
