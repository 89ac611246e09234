"""Key metrics of every launch in an .ncu-rep (`ncu --set full` capture) as a small CSV for profiles/.

    python scripts/ncu_summary.py measure_out/X.ncu-rep > profiles/X.csv
"""
import csv, subprocess, sys

KEYS = ["ID", "Kernel Name", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "gpu__time_duration.sum",
        "smsp__inst_executed.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.avg.per_cycle_active",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum",
        "lts__t_sector_hit_rate.pct", "l1tex__t_bytes.sum", "smsp__cycles_active.avg", "sm__cycles_elapsed.max",
        "launch__shared_mem_per_block_static", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_warps", "sm__maximum_warps_per_active_cycle_pct"]

raw = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True, check=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]
cols = [hdr.index(k) for k in KEYS if k in hdr]
w = csv.writer(sys.stdout)
w.writerow([hdr[i] for i in cols])
w.writerow([units[i] for i in cols])
for r in rows[2:]:
    w.writerow([r[i] for i in cols])
