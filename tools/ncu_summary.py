"""Summarise an `ncu --set full` report (read here, on the CPU box): per captured launch the duration, DRAM bytes read/written,
DRAM / SM throughput, issue-active, registers.   python tools/ncu_summary.py report.ncu-rep [algorithmic_bytes]"""
import csv
import io
import subprocess
import sys


def main():
    rep = sys.argv[1]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, body = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}

    def pick(*names):
        for n in names:
            for h in hdr:
                if h == n or h.endswith(n):
                    return col[h]
        return None

    keys = [("kernel", pick("Kernel Name")), ("grid", pick("Grid Size")), ("block", pick("Block Size")), ("time", pick("gpu__time_duration.sum")),
            ("dram_rd", pick("dram__bytes_read.sum")), ("dram_wr", pick("dram__bytes_write.sum")),
            ("dram_pct", pick("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed")), ("sm_pct", pick("sm__throughput.avg.pct_of_peak_sustained_elapsed")),
            ("issue_active_pct", pick("smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_issued.avg.pct_of_peak_sustained_active")),
            ("regs", pick("launch__registers_per_thread")), ("smem_conflict", pick("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum")),
            ("warps_active_pct", pick("sm__warps_active.avg.pct_of_peak_sustained_active"))]
    for r in body:
        out = {}
        for k, i in keys:
            if i is not None and i < len(r):
                out[k] = "%s %s" % (r[i], units[i]) if units[i] else r[i]
        print(out)


if __name__ == "__main__":
    main()
