"""Turn .ncu-rep captures into text summaries under profiles/ (generated locally, not committed)."""
import csv
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "dram_read"),
    ("dram__bytes_write.sum", "dram_write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "l2_pct"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm_pct"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor_pipe_pct"),
    ("sm__inst_executed_pipe_tensor.sum", "tensor_inst"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps_active_pct"),
    ("launch__registers_per_thread", "regs"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__shared_mem_per_block_dynamic", "dyn_smem"),
    ("smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "stall_long_sb"),
    ("l1tex__t_sector_hit_rate.pct", "l1_hit"),
    ("lts__t_sector_hit_rate.pct", "l2_hit"),
]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    with open(out, "w") as fh:
        fh.write(f"# ncu --set full summary of {rep.split('/')[-1]} (ncu -i ... --page raw --csv)\n")
        for row in rows[2:]:
            name = row[hdr.index("Kernel Name")]
            fh.write(f"\n## {name[:110]}\n")
            for key, label in KEYS:
                # tolerate metric-name variants
                idx = [i for i, h in enumerate(hdr) if h == key]
                if idx:
                    fh.write(f"{label:>18}: {row[idx[0]]} {units[idx[0]]}\n")
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
