"""Turns one `ncu --set full --import-source on` capture of the fused kernel into evidence files (kept out of git):
  profiles/<tag>_ncu_full_summary.json   key metrics of the captured launch
  profiles/<tag>_ncu_raw.csv             the full --page raw export
  profiles/<tag>_source_hotspots.txt     warp-stall samples and executed instructions per CUDA source line (top 40)
  profiles/traffic.json                  dram bytes per launch, tied to the sha of the kernel sources (bench.py reads it)
usage: python scripts/ncu_summarise.py <capture>.ncu-rep <tag> [workload-key]"""
import csv, io, json, os, subprocess, sys, collections

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
rep, tag = sys.argv[1], sys.argv[2]
key = sys.argv[3] if len(sys.argv) > 3 else "c4"
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
open(os.path.join(ROOT, "profiles", f"{tag}_ncu_raw.csv"), "w").write(raw)
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, vals = rows[0], rows[1], rows[2]
col = {h: i for i, h in enumerate(hdr)}
keep = ["Kernel Name", "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "dram__bytes_read.sum", "dram__bytes_write.sum", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct"]
keep += [h for h in hdr if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
summary = {h: (vals[col[h]] + " " + units[col[h]]).strip() for h in keep if h in col}
json.dump(summary, open(os.path.join(ROOT, "profiles", f"{tag}_ncu_full_summary.json"), "w"), indent=1)


def to_bytes(h):
    v, u = float(vals[col[h]]), units[col[h]].lower()
    return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}[u]


import bench  # source_sha
traffic = to_bytes("dram__bytes_read.sum") + to_bytes("dram__bytes_write.sum")
tj_path = os.path.join(ROOT, "profiles", "traffic.json")
tj = {}
if os.path.exists(tj_path):
    tj = json.load(open(tj_path))
    if tj.get("source_sha") != bench.source_sha():
        tj = {}
tj[key] = traffic
tj["source_sha"] = bench.source_sha()
tj["note"] = (f"dram__bytes_read.sum + dram__bytes_write.sum of one {summary.get('Kernel Name')} launch "
              f"(ncu --set full, cold L2), profiles/{tag}_ncu_full_summary.json")
json.dump(tj, open(tj_path, "w"), indent=1)

src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass,cuda"], capture_output=True, text=True).stdout
per = collections.OrderedDict()
cur_file = None
reader = csv.reader(io.StringIO(src))
head = None
for r in reader:
    if not r:
        continue
    if r[0] == "File Path":
        cur_file = os.path.basename(r[1]); continue
    if r[0] == "Function Name":
        continue
    if r[0] == "Line No":
        head = {h: i for i, h in enumerate(r)}; continue
    if head is None or not r[0]:
        continue  # SASS rows have an empty line number
    try:
        line = int(r[0])
    except ValueError:
        continue
    def num(x):
        try:
            return int(x)
        except ValueError:
            return 0
    samples = num(r[head["# Samples"]])
    inst = num(r[head["Instructions Executed"]])
    k = (cur_file, line)
    s0, i0, t0 = per.get(k, (0, 0, r[1]))
    per[k] = (s0 + samples, i0 + inst, r[1])
total = sum(v[0] for v in per.values()) or 1
total_inst = sum(v[1] for v in per.values()) or 1
with open(os.path.join(ROOT, "profiles", f"{tag}_source_hotspots.txt"), "w") as f:
    f.write(f"# {summary.get('Kernel Name')}: warp stall samples and executed warp instructions by CUDA source line\n")
    f.write(f"# total samples {total}, total warp instructions {total_inst}; share of samples | share of instructions | file:line | source\n")
    for (fn, ln), (s, i, text) in sorted(per.items(), key=lambda kv: -kv[1][0])[:40]:
        f.write(f"{100.0*s/total:5.1f}% | {100.0*i/total_inst:5.1f}% | {fn}:{ln} | {text.strip()[:110]}\n")
print(json.dumps(summary, indent=1)[:600])
print("traffic", traffic)
