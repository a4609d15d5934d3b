"""summarise an .ncu-rep (ncu --set full) into per-kernel figures (one JSON object per kernel):
python tools/ncu_summary.py <report.ncu-rep> [command string] > summary.json"""
import csv, io, json, subprocess, sys
rep = sys.argv[1]
cmd = sys.argv[2] if len(sys.argv) > 2 else ""
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
want = {"gpu__time_duration.sum": "duration", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active": "tensor_pipe_active_pct",
        "sm__warps_active.avg.pct_of_peak_sustained_active": "warps_active_pct", "dram__bytes_read.sum": "dram_read", "dram__bytes_write.sum": "dram_write",
        "launch__registers_per_thread": "registers_per_thread", "lts__t_sector_hit_rate.pct": "l2_hit_pct", "l1tex__t_sector_hit_rate.pct": "l1_hit_pct",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed": "sm_throughput_pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed": "l2_throughput_pct",
        "sm__inst_issued.avg.pct_of_peak_sustained_active": "issue_active_pct", "launch__grid_size": "grid", "launch__block_size": "block",
        "launch__shared_mem_per_block_dynamic": "dyn_smem", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed": "dram_throughput_pct",
        "smsp__inst_executed.sum": "smsp_inst"}
idx = {n: i for i, n in enumerate(hdr)}
out = []
for r in rows[2:]:
    if len(r) < len(hdr): continue
    e = {"kernel": r[idx["Kernel Name"]], "report": rep.split("/")[-1], "command": cmd}
    for m, k in want.items():
        if m in idx: e[k] = f"{r[idx[m]]} {units[idx[m]]}".strip()
    out.append(e)
print(json.dumps({"how": "ncu --set full --clock-control none --import-source on (values per launch; read with ncu -i <rep> --page raw --csv)", "kernels": out}, indent=1))
