"""Compact summary of an `ncu --set full` report (written under profiles/, which git ignores).  Usage: python tools/ncu_summary.py report.ncu-rep [more.ncu-rep ...] > profiles/rN_ncu_<what>.md"""
import csv
import io
import json
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "duration"),
    ("sm__cycles_elapsed.avg", "SM cycles elapsed (avg)"),
    ("sm__cycles_active.avg", "SM cycles active (avg)"),
    ("sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe busy, % of ACTIVE cycles"),
    ("sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor pipe busy, % of ELAPSED cycles"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput %"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate %"),
    ("lts__t_bytes.sum", "L2 traffic"),
    ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "LSU shared-memory wavefronts"),
    ("l1tex__t_requests_pipe_lsu_mem_global_op_st.sum", "global store requests"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum", "global store sectors"),
    ("l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum", "global load requests"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "global load sectors"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__registers_per_thread", "registers / thread"),
    ("launch__shared_mem_per_block_dynamic", "dynamic smem / block"),
    ("smsp__inst_executed.sum", "warp instructions executed"),
]


def rows_of(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    return [(dict(zip(hdr, r)), dict(zip(hdr, units))) for r in rows[2:]]


def main():
    for rep in sys.argv[1:]:
        for vals, units in rows_of(rep):
            print("## %s  --  %s" % (rep.split("/")[-1], vals.get("Kernel Name", "?")))
            print()
            print("| metric | value |")
            print("|---|---|")
            d = {}
            for key, label in WANT:
                if key in vals:
                    print("| %s (`%s`) | %s %s |" % (label, key, vals[key], units.get(key, "")))
                    d[key] = vals[key]
            try:
                act = float(d["sm__cycles_active.avg"].replace(",", ""))
                el = float(d["sm__cycles_elapsed.avg"].replace(",", ""))
                print("| SM active / elapsed | %.3f |" % (act / el))
            except Exception:
                pass
            try:
                scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
                tscale = {"ns": 1e-9, "us": 1e-6, "ms": 1e-3, "s": 1.0}
                by = sum(float(d[k].replace(",", "")) * scale[units[k]] for k in ("dram__bytes_read.sum", "dram__bytes_write.sum"))
                t = float(d["gpu__time_duration.sum"].replace(",", "")) * tscale[units["gpu__time_duration.sum"]]
                print("| achieved HBM GB/s ((read + write) / duration) | %.0f |" % (by / t / 1e9))
            except Exception:
                pass
            print()


if __name__ == "__main__":
    main()
