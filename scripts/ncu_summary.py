"""Summarises an .ncu-rep (raw + SASS source pages) into a small text report on stdout."""
import collections, csv, subprocess, sys, io
rep = sys.argv[1]; frames = int(sys.argv[2]) if len(sys.argv) > 2 else 512000
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw))); hdr, units, data = rows[0], rows[1], rows[2:]
want = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed.avg.per_cycle_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__grid_size", "launch__block_size",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__warps_active.avg.per_cycle_active", "smsp__warps_eligible.avg.per_cycle_active", "sm__cycles_elapsed.avg",
        "smsp__average_warp_latency_per_inst_issued.ratio"]
print(f"# ncu summary of {rep} ({frames} frames per launch)")
for w in want:
    if w in hdr:
        i = hdr.index(w); print(f"{w:75s} {units[i]:14s} {[r[i] for r in data]}")
stalls = [(h, float(data[0][i])) for i, h in enumerate(hdr) if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
print("\n# warp stall reasons (warps stalled per issue-active cycle)")
for h, v in sorted(stalls, key=lambda x: -x[1])[:10]:
    print(f"{h[len('smsp__average_warps_issue_stalled_'):-len('_per_issue_active.ratio')]:28s} {v:.3f}")
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(src)))
hi = [i for i, r in enumerate(rows) if r and r[0] == "Address"]
h = rows[hi[0]]; body = rows[hi[0] + 1:(hi[1] - 1 if len(hi) > 1 else len(rows))]
ci, si = h.index("Instructions Executed"), h.index("Source")
ws, wsi = h.index("L1 Wavefronts Shared"), h.index("L1 Wavefronts Shared Ideal")
tot = 0; byop = collections.Counter(); wav = collections.Counter(); wavi = collections.Counter()
for r in body:
    try: n = int(r[ci])
    except Exception: continue
    t = r[si].strip().split()
    if not t: continue
    o = t[1] if t[0].startswith("@") else t[0]
    parts = o.split(".")
    o = parts[0] + ("." + parts[1] if parts[0] in ("LDS", "STS", "LDG", "STG", "SHFL") and len(parts) > 1 else "")
    tot += n; byop[o] += n; wav[o] += int(r[ws] or 0); wavi[o] += int(r[wsi] or 0)
print(f"\n# SASS mix: {tot} warp instructions, {tot / frames:.1f} per frame, {2 * tot / frames:.1f} per lane-frame (half-warp per frame)")
for o, n in byop.most_common(28):
    extra = f" smem wavefronts {wav[o]} (ideal {wavi[o]})" if wav[o] else ""
    print(f"{o:12s} {n:12d} {100 * n / tot:5.1f}%  {2 * n / frames:7.1f}/lane-frame{extra}")
