"""Turns `ncu --set full` reports into markdown tables (runs without a GPU: `ncu -i <rep> --page raw --csv`).

    python scripts/ncu_summary.py <title> <report.ncu-rep> [<report2.ncu-rep> ...] > ncu_summary_<name>.md
    python scripts/ncu_summary.py --traffic <report.ncu-rep> > traffic.json
"""
import csv
import io
import json
import subprocess
import sys

METRICS = [
    "gpu__time_duration.sum",
    "dram__bytes_read.sum",
    "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "launch__registers_per_thread",
    "launch__block_size",
    "launch__grid_size",
    "launch__shared_mem_per_block_dynamic",
    "launch__shared_mem_config_size",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum",
    "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed",
    "l1tex__t_sector_hit_rate.pct",
    "lts__t_sector_hit_rate.pct",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_red.sum",
    "lts__t_sectors_srcunit_tex_op_read.sum",
    "lts__t_sectors_srcunit_tex_op_red.sum",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
    "sm__cycles_elapsed.max",
]


def rows_of(report):
    out = subprocess.run(["ncu", "-i", report, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    return hdr, units, rows[2:]


def main():
    if sys.argv[1] == "--traffic":
        hdr, units, rows = rows_of(sys.argv[2])
        r = rows[0]

        def val(name):
            i = hdr.index(name)
            v = float(r[i].replace(",", ""))
            return v * {"Mbyte": 1e6, "Kbyte": 1e3, "Gbyte": 1e9, "byte": 1.0}[units[i]]

        print(json.dumps({"kernel": r[hdr.index("Kernel Name")], "dram_bytes_read_per_launch": int(val("dram__bytes_read.sum")), "dram_bytes_write_per_launch": int(val("dram__bytes_write.sum")),
                          "source": f"ncu --set full --clock-control none ({sys.argv[2].split('/')[-1]}); dram__bytes_read.sum + dram__bytes_write.sum"}, indent=1))
        return
    print(f"# {sys.argv[1]}\n")
    print("Captured with `ncu --set full --clock-control none --import-source on`; read with `ncu -i … --page raw --csv`")
    print("(scripts/ncu_summary.py). Times under ncu are serialised / cold-cache: bench numbers come from bench.py / scripts/bench_mlp.py only.\n")
    for rep in sys.argv[2:]:
        hdr, units, rows = rows_of(rep)
        for r in rows:
            print(f"## `{r[hdr.index('Kernel Name')]}`  ({rep.split('/')[-1]})\n")
            print("| metric | unit | value |\n|---|---|---|")
            for m in METRICS:
                if m in hdr:
                    i = hdr.index(m)
                    print(f"| `{m}` | {units[i]} | {r[i]} |")
            print()


if __name__ == "__main__":
    main()
