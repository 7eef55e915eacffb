"""Turns the ncu captures of a round (gpurun_out/rN_launches.csv, gpurun_out/rN_full.ncu-rep, gpurun_out/rN_bench*.json) into the tracked
summaries under profiles/.  Usage: python scripts/summarize_profiles.py r1"""
import csv, json, os, subprocess, sys, collections

tag = sys.argv[1] if len(sys.argv) > 1 else "r1"
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
go, pr = os.path.join(root, "gpurun_out"), os.path.join(root, "profiles")


def last_json(path):
    return json.loads([l for l in open(path).read().splitlines() if l.startswith("{")][-1])


# ---- launch list -------------------------------------------------------------------------------------------------------------------------
rows = [r for r in csv.reader(open(os.path.join(go, tag + "_launches.csv"))) if len(r) > 5]
h = [i for i, r in enumerate(rows) if r[0] == "ID"][0]
H, data = rows[h], rows[h + 1:]
ki, vi, ui = H.index("Kernel Name"), H.index("Metric Value"), H.index("Metric Unit")
frames, cur = [], None
for r in data:
    name = r[ki].split("(")[0].replace("void pt::", "").replace("pt::", "").replace("void ", "")
    t = float(r[vi].replace(",", "")) * {"ns": 1e-6, "us": 1e-3, "ms": 1.0}[r[ui]]
    if name.startswith("k_generate"): cur = []; frames.append(cur)
    if cur is not None: cur.append((name, t))
frame = frames[3]                      # first timed frame after 3 warm-up frames
per = collections.OrderedDict(); cnt = collections.Counter()
for n, t in frame: per[n] = per.get(n, 0.0) + t; cnt[n] += 1
total = sum(per.values())
open(os.path.join(pr, tag + "_ncu_launches.csv"), "w").write(open(os.path.join(go, tag + "_launches.csv")).read())

# ---- full capture ------------------------------------------------------------------------------------------------------------------------
raw = subprocess.run(["ncu", "-i", os.path.join(go, tag + "_full.ncu-rep"), "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rr = list(csv.reader(raw.splitlines())); hdr, units, drows = rr[0], rr[1], rr[2:]
want = [("Kernel Name", "kernel"), ("gpu__time_duration.sum", "time"), ("dram__bytes_read.sum", "dram_read"), ("dram__bytes_write.sum", "dram_write"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct"), ("lts__t_sector_hit_rate.pct", "l2_hit_pct"), ("l1tex__t_sector_hit_rate.pct", "l1_hit_pct"),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "occupancy_pct"), ("launch__registers_per_thread", "regs"),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue_active_pct"), ("smsp__thread_inst_executed_per_inst_executed.ratio", "threads_per_inst"),
        ("smsp__inst_executed.sum", "warp_insts"), ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "pipe_alu_pct"),
        ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "pipe_fma_pct"), ("sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "pipe_xu_pct"),
        ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "pipe_lsu_pct"),
        ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall_long_scoreboard"), ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall_wait")]
full = []
for r in drows:
    d = {}
    for hname, k in want:
        if hname not in hdr: continue
        i = hdr.index(hname); v, u = r[i], units[i]
        if k in ("dram_read", "dram_write"): d[k + "_bytes"] = float(v) * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[u]
        elif k == "time": d["time_ms"] = float(v) * {"us": 1e-3, "ms": 1, "ns": 1e-6, "s": 1e3}.get(u, 1)
        elif k == "kernel": d[k] = v.split("(")[0].replace("void pt::", "").replace("void ", "")
        else:
            try: d[k] = float(v)
            except ValueError: d[k] = v
    full.append(d)
json.dump(full, open(os.path.join(pr, tag + "_ncu_full_summary.json"), "w"), indent=1)

# ---- bench lines ---------------------------------------------------------------------------------------------------------------------------
b = last_json(os.path.join(go, tag + "_bench.json"))
json.dump(b, open(os.path.join(pr, tag + "_bench_n1.json"), "w"))
if os.path.exists(os.path.join(go, tag + "_bench_reference.json")):
    json.dump(last_json(os.path.join(go, tag + "_bench_reference.json")), open(os.path.join(pr, tag + "_bench_reference_n1.json"), "w"))
km = b["roofline"]["kernel_ms_per_frame"]; tot_b = sum(km.values())

md = ["# Round %s profiles (sm_90a, default build)\n" % tag[1:],
      "Workload = `bench.py` default: %s\n" % b["config"]["workload"],
      "Bench line (`%s_bench_n1.json`): **%.0f Mrays/s, %.2f ms/frame** device-resident, e2e %.0f Mrays/s, roofline.frac %.3f (algorithmic %.0f GB/s of %.0f GB/s measured peak), "
      "ncu DRAM traffic of the traversal kernel %.2f GB/frame vs %.1f GB algorithmic.\n" % (tag, b["value"], b["ms_per_step"], b["e2e"]["value"], b["roofline"]["frac"], b["roofline"]["achieved"],
                                                                                              b["roofline"]["peak"], (b["roofline"]["traffic"] or 0) / 1e9, b["roofline"]["algorithmic_bytes_per_frame"] / 1e9),
      "## 1. Launch list (`%s_ncu_launches.csv`)\n" % tag,
      "`ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline`; first timed frame (%d launches), serialised / cold-cache times; "
      "shares compared with the CUDA-event shares of the bench line's timing context:\n" % len(frame),
      "| kernel | launches | ncu ms | ncu share | bench (events) ms | bench share |\n|---|---|---|---|---|---|"]
mp = {"k_trace_closest": "trace_closest", "k_shade": "shade", "k_trace_shadow": "trace_shadow"}
other = 0.0
for n, t in per.items():
    key = [v for k, v in mp.items() if n.startswith(k)]
    if key: md.append("| %s | %d | %.3f | %.1f %% | %.3f | %.1f %% |" % (n, cnt[n], t, 100 * t / total, km[key[0]], 100 * km[key[0]] / tot_b))
    else: other += t
md.append("| k_generate + k_commit_accumulate | 2 | %.3f | %.1f %% | %.3f | %.1f %% |" % (other, 100 * other / total, km["other"], 100 * km["other"] / tot_b))
md.append("| frame | %d | %.3f | | %.3f serialised (measured frame with shadow/closest overlap: %.3f) | |\n" % (len(frame), total, tot_b, b["ms_per_step"]))
md.append("## 2. `ncu --set full` of the three wavefront kernels, iterations 0..2 of one frame (`%s_ncu_full_summary.json`)\n" % tag)
md.append("`ncu --set full --clock-control none --import-source on -k regex:\"k_trace_closest|k_shade|k_trace_shadow\" -s 99 -c 9 python bench.py --steps 1 --warmup 3 --no-cpu-baseline`\n")
md.append("| # | kernel | ms | DRAM rd MB | DRAM wr MB | DRAM % peak | L2 hit % | L1 hit % | occupancy % | regs | issue active % | threads/inst | warp inst (M) | ALU % | FMA % | XU % | LSU % | long-scoreboard | wait |\n" + "|---" * 19 + "|")
for i, d in enumerate(full):
    md.append("| %d | %s | %.3f | %.0f | %.0f | %.1f | %.1f | %.1f | %.1f | %d | %.1f | %.1f | %.0f | %.1f | %.1f | %.1f | %.1f | %.2f | %.2f |" % (
        i, d["kernel"], d["time_ms"], d["dram_read_bytes"] / 1e6, d["dram_write_bytes"] / 1e6, d["dram_pct"], d["l2_hit_pct"], d["l1_hit_pct"], d["occupancy_pct"], d["regs"], d["issue_active_pct"],
        d["threads_per_inst"], d["warp_insts"] / 1e6, d.get("pipe_alu_pct", 0), d.get("pipe_fma_pct", 0), d.get("pipe_xu_pct", 0), d.get("pipe_lsu_pct", 0), d.get("stall_long_scoreboard", 0), d.get("stall_wait", 0)))
md.append(open(os.path.join(pr, tag + "_reading.md")).read() if os.path.exists(os.path.join(pr, tag + "_reading.md")) else "")
open(os.path.join(pr, tag + "_summary.md"), "w").write("\n".join(md))
print("\n".join(md[-14:]))
