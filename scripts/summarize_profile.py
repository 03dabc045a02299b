"""Summarise the ncu captures of scripts/collect_profiles.sh into profiles/ (per-GPU summaries, not kept in git): python scripts/summarize_profile.py r01"""
import csv, json, os, subprocess, sys
tag = sys.argv[1] if len(sys.argv) > 1 else "r01"
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
go, pr = os.path.join(root, "gpurun_out"), os.path.join(root, "profiles")
os.makedirs(pr, exist_ok=True)
# ---- launch list
lp = os.path.join(go, f"{tag}_launches.csv")
if os.path.exists(lp):
    rows = [r for r in csv.reader(l for l in open(lp) if not l.startswith("=="))]
    hdr = rows[0]; ki = hdr.index("Kernel Name"); vi = hdr.index("Metric Value"); ui = hdr.index("Metric Unit")
    agg = {}
    for r in rows[1:]:
        if len(r) <= vi: continue
        v = float(r[vi].replace(",", "")); u = r[ui]
        ms = v / 1e6 if u in ("ns", "nsecond") else (v / 1e3 if u in ("us", "usecond") else v)
        a = agg.setdefault(r[ki][:110], [0, 0.0]); a[0] += 1; a[1] += ms
    tot = sum(a[1] for a in agg.values())
    with open(os.path.join(pr, f"{tag}_launches.md"), "w") as f:
        f.write(f"# {tag}: every kernel launched by `python bench.py --steps 2 --warmup 1 --no-cpu` under ncu (gpu__time_duration.sum, --clock-control none)\n\n")
        f.write("Per-launch times under ncu are cold-cache and serialised: compare SHARES, not absolutes.\n\n| kernel | launches | total ms | share |\n|---|---|---|---|\n")
        for k, a in sorted(agg.items(), key=lambda x: -x[1][1]):
            f.write(f"| `{k}` | {a[0]} | {a[1]:.3f} | {100*a[1]/tot:.1f}% |\n")
    print(open(os.path.join(pr, f"{tag}_launches.md")).read())
# ---- full capture
rep = os.path.join(go, f"{tag}_full.ncu-rep")
if os.path.exists(rep):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, unit, val = rows[0], rows[1], rows[2]
    want = ["Kernel Name", "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
            "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.per_cycle_active",
            "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
            "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
            "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__issue_active.avg.pct_of_peak_sustained_elapsed",
            "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
            "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum", "sm__icc_request_hit_rate.pct",
            "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
            "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
            "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
            "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum"]
    out = {}
    with open(os.path.join(pr, f"{tag}_ncu_capture_table.md"), "w") as f:
        f.write(f"# {tag}: `ncu --set full --clock-control none --import-source on` of the kernel scripts/collect_profiles.sh selected\n\n| metric | unit | value |\n|---|---|---|\n")
        for w in want:
            if w in hdr:
                i = hdr.index(w); f.write(f"| {w} | {unit[i]} | {val[i]} |\n"); out[w] = (unit[i], val[i])
    def tobytes(u, v):
        v = float(v.replace(",", ""))
        return v * {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1, "Tbyte": 1e12}.get(u, 1)
    if "dram__bytes_read.sum" in out:
        tr = tobytes(*out["dram__bytes_read.sum"]) + tobytes(*out["dram__bytes_write.sum"])
        print("dram bytes per launch", tr)
    print(open(os.path.join(pr, f"{tag}_ncu_capture_table.md")).read())
