"""Summarise an .ncu-rep (ncu --set full) into the handful of metrics DESIGN.md / bench.py quote.
usage: python profiles/summarize_ncu.py /tmp/prof.ncu-rep > <name>.md"""
import csv
import io
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.sum", "sm__cycles_active.avg", "sm__cycles_elapsed.max",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__cycles_active.avg",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
        "launch__block_size", "launch__shared_mem_per_block_dynamic", "sm__maximum_warps_per_active_cycle_pct",
        "smsp__inst_executed.sum", "l1tex__m_xbar2l1tex_read_bytes.sum", "sm__sass_inst_executed_op_shared_ld.sum",
        "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct", "sm__mio_inst_issued.sum",
        "smsp__average_warps_issue_stalled", "smsp__issue_active.avg.pct", "smsp__inst_executed_pipe_fma",
        "sm__pipe_fma_cycles_active.avg.pct", "sm__inst_executed_pipe_lsu", "smsp__inst_executed_pipe_fmaheavy",
        "sm__pipe_fmaheavy_cycles_active.avg.pct", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared",
        "smsp__inst_executed_op_shared", "sm__warps_active.avg.per_cycle_active", "smsp__inst_issued.avg.per_cycle_active"]


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    if len(rows) < 3:
        print("no data in", path)
        return
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    print("# ncu summary of `%s`\n" % path)
    for r in rows[2:]:
        name = r[idx["Kernel Name"]][:70]
        print("## %s  (id %s, grid %s, block %s)\n" % (name, r[idx["ID"]], r[idx.get("Grid Size", 0)], r[idx.get("Block Size", 0)]))
        print("| metric | value | unit |\n|---|---|---|")
        for k in hdr:
            if any(k.startswith(p) for p in KEYS) or "tensor" in k and "pct" in k or k.startswith("smsp__average_warps_issue_stalled") and "pct" not in k and False:
                v = r[idx[k]]
                if v not in ("", "n/a"):
                    print("| %s | %s | %s |" % (k, v, units[idx[k]]))
        print()


if __name__ == "__main__":
    main(sys.argv[1])
