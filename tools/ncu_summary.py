#!/usr/bin/env python
"""Turn an `ncu --set full` report into a short text summary.

    python tools/ncu_summary.py prof.ncu-rep [--samples N --bytes-per-sample B] > ncu_summary.txt

Reads the report with `ncu -i <rep> --page raw --csv` (no GPU needed) and prints, per captured launch, the metrics the
roofline discussion in DESIGN.md uses: duration, DRAM bytes read / written (the `traffic` of bench.py's roofline object),
DRAM and SM throughput, issue activity, occupancy, registers, pipe utilisation, instruction count (per sample if --samples)."""
import argparse
import csv
import io
import subprocess
import sys

WANT = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__occupancy_limit_registers", "launch__grid_size", "launch__block_size",
    "smsp__inst_executed.sum", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum", "lts__t_sector_hit_rate.pct",
]


def to_bytes(value, unit):
    v = float(value.replace(",", ""))
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}.get(unit, 1)


def to_seconds(value, unit):
    v = float(value.replace(",", ""))
    return v * {"ns": 1e-9, "us": 1e-6, "ms": 1e-3, "s": 1.0}.get(unit, 1e-9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("report")
    ap.add_argument("--samples", type=float, default=0, help="samples one launch processes (for per-sample figures)")
    ap.add_argument("--bytes-per-sample", type=float, default=0, help="algorithmic bytes per sample (SURVEY 8d)")
    ap.add_argument("--peak-gbs", type=float, default=3350.0, help="HBM peak (default: H100 SXM data sheet)")
    ap.add_argument("--traffic-json", default="", help="also write the DRAM bytes per sample of the demodulation kernels (bench.py's "
                    "roofline.traffic): {detect: k_fsk_fifo<WRITE,STATS>, given: k_fsk_fifo<DIGITIZE,WRITE>}; needs --samples")
    ap.add_argument("--capture-note", default="", help="where the capture is summarised (recorded in the traffic file)")
    args = ap.parse_args()
    raw = subprocess.run(["ncu", "-i", args.report, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}
    print("source: %s (ncu --page raw)" % args.report)
    traffic = {}
    for d in data:
        print("\n== " + d[col["Kernel Name"]][:150])
        for w in WANT:
            if w in col:
                print("  %-72s %s %s" % (w, d[col[w]], units[col[w]]))
        try:
            t = to_seconds(d[col["gpu__time_duration.sum"]], units[col["gpu__time_duration.sum"]])
            rd = to_bytes(d[col["dram__bytes_read.sum"]], units[col["dram__bytes_read.sum"]])
            wr = to_bytes(d[col["dram__bytes_write.sum"]], units[col["dram__bytes_write.sum"]])
            print("  %-72s %.1f GB/s (%.1f %% of %.1f)" % ("derived: DRAM traffic / duration", (rd + wr) / t / 1e9, 100 * (rd + wr) / t / 1e9 / args.peak_gbs, args.peak_gbs))
            name = d[col["Kernel Name"]]
            if args.samples and "k_fsk_fifo<4, 0, 1, 1>" in name:
                traffic["detect"] = {"kernel": "k_fsk_fifo<F32,WRITE,STATS>", "dram_bytes_per_sample": (rd + wr) / args.samples, "capture": args.capture_note}
            if args.samples and "k_fsk_fifo<4, 1, 1, 0>" in name:
                traffic["given"] = {"kernel": "k_fsk_fifo<F32,DIGITIZE,WRITE>", "dram_bytes_per_sample": (rd + wr) / args.samples, "capture": args.capture_note}
            if args.samples and args.bytes_per_sample:
                alg = args.samples * args.bytes_per_sample
                print("  %-72s %.3f GB -> %.1f GB/s (%.1f %%); DRAM traffic / algorithmic = %.3f" % (
                    "derived: algorithmic bytes", alg / 1e9, alg / t / 1e9, 100 * alg / t / 1e9 / args.peak_gbs, (rd + wr) / alg))
            if args.samples and "smsp__inst_executed.sum" in col:
                inst = float(d[col["smsp__inst_executed.sum"]].replace(",", ""))
                print("  %-72s %.1f" % ("derived: thread instructions per sample", inst * 32 / args.samples))
        except (KeyError, ValueError, ZeroDivisionError):
            pass
    if args.traffic_json and traffic:
        import json

        with open(args.traffic_json, "w") as fh:
            json.dump(traffic, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
