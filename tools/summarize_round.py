"""Turn the gpurun_out/ of `bash tools/gpu_round.sh all` into committed artefacts under profiles/<tag>_*.

    python tools/summarize_round.py r01e

Copies the bench lines, test / sanitizer logs and the ncu launch list, exports the first captured launch of each
`ncu --set full` report as raw CSV, aggregates the source page per line / function and writes <tag>_SUMMARY.md."""
import collections
import csv
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT, PROF = os.path.join(ROOT, "gpurun_out"), os.path.join(ROOT, "profiles")
tag = sys.argv[1]


def cp(src, dst):
    s = os.path.join(OUT, src)
    if os.path.exists(s):
        shutil.copy(s, os.path.join(PROF, "%s_%s" % (tag, dst)))
        return True
    return False


for src, dst in [("bench.json", "bench_c2.json"), ("bench_ref.json", "bench_reference_arm.json"),
                 ("bench_c3.json", "bench_c3.json"), ("bench_c4.json", "bench_c4_covid.json"),
                 ("bench_c5.json", "bench_c5.json"), ("pytest_gpu.log", "pytest_gpu.log"),
                 ("racecheck.log", "racecheck.log"), ("memcheck.log", "memcheck.log"),
                 ("launches.csv", "launches_c2.csv"), ("smoke.log", "smoke.log")]:
    cp(src, dst)

raw = {}
for rep, name in [("prof_step.ncu-rep", "aie_step_kernel"), ("prof_observe.ncu-rep", "aie_observe_kernel")]:
    path = os.path.join(OUT, rep)
    if not os.path.exists(path):
        continue
    txt = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    with open(os.path.join(PROF, "%s_ncu_full_%s_raw.csv" % (tag, name)), "w", newline="") as f:
        w = csv.writer(f)
        for r in rows[:3]:
            w.writerow(r)
    raw[name] = (dict(zip(rows[0], rows[2])), dict(zip(rows[0], rows[1])), len(rows) - 2)

# per-line / per-function split of the step kernel (first launch's sections only)
rep = os.path.join(OUT, "prof_step.ncu-rep")
if os.path.exists(rep):
    txt = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"],
                         capture_output=True, text=True).stdout.splitlines()
    first = None
    for i, line in enumerate(txt):
        if line.startswith('"File Path"'):
            if first is None:
                first = line
            elif line == first:
                txt = txt[:i]
                break
    tmp = "/tmp/%s_src.csv" % tag
    open(tmp, "w").write("\n".join(txt))
    n_launch = raw.get("aie_step_kernel", (None, None, 1))[2]
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_by_line.py"), tmp, str(8192 * n_launch), "60"],
                         capture_output=True, text=True, cwd=ROOT).stdout
    with open(os.path.join(PROF, "%s_step_kernel_by_line.txt" % tag), "w") as f:
        f.write("# ncu --set full source page (cuda,sass) of the fused step kernel, workload c2; samples and instruction counts are "
                "summed over the %d captured launches (per-env figures divided by %d x 8192 envs); lines of inlined callees are "
                "also counted under their call sites (about 10 %% overlap).\n" % (n_launch, n_launch))
        f.write("\n".join(l[:220] for l in res.splitlines()))

# launch list shares
shares = []
lp = os.path.join(OUT, "launches.csv")
if os.path.exists(lp):
    rows = list(csv.reader(open(lp)))
    h = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    ki, vi = rows[h].index("Kernel Name"), rows[h].index("Metric Value")
    agg = collections.defaultdict(list)
    for r in rows[h + 2:]:
        if len(r) > vi:
            try:
                agg[r[ki].split("(")[0]].append(float(r[vi].replace(",", "")))
            except ValueError:
                pass
    tot = sum(sum(v) for v in agg.values())
    unit = 1e3 if max(max(v) for v in agg.values()) > 1e4 else 1.0
    shares = [(k, len(v), sum(v) / len(v) / unit, 100 * sum(v) / tot) for k, v in agg.items()]

b = json.load(open(os.path.join(OUT, "bench.json")))
k = b["roofline"]["kernels"]
lines = ["# Round 1 (%s) — H100 measurements, workload c2 (4 agents, 25x25, 8192 env replicas, 1 GPU)" % tag[-1], "",
         "Command: `bash tools/gpu_round.sh all` under gpurun; artefacts copied by `tools/summarize_round.py %s`." % tag, "",
         "## bench.py (CUDA events, %d steps after %d warm-up)" % (b["steps"], b["warmup"]), "",
         "* value = %.3e agent-env-steps/s (%.4f ms per step of 8192 envs); e2e (all outputs to pinned host) = %.3e"
         % (b["value"], b["ms_per_step"], b["e2e"]["value"]),
         "* whole-step algorithmic bytes = %d B/env-step -> %.0f GB/s = %.3f of the measured HBM peak (%.1f GB/s)"
         % (b["roofline"]["whole_step"]["alg_bytes_per_env_step"], b["roofline"]["whole_step"]["achieved"],
            b["roofline"]["whole_step"]["frac"], b["roofline"]["peak"]),
         "* aie_step_kernel: %.1f us/launch, %.0f GB/s algorithmic, frac %.3f; unfused legs: dynamics only %.1f us, observe only %.1f us"
         % (k["aie_step_kernel"]["ms"] * 1e3, k["aie_step_kernel"]["achieved_gbs"], k["aie_step_kernel"]["frac"],
            k["aie_step_kernel"]["unfused_ms"]["dynamics_only"] * 1e3, k["aie_step_kernel"]["unfused_ms"]["observe_only"] * 1e3),
         "* aie_sample_kernel: %.1f us/launch" % (k["aie_sample_kernel"]["ms"] * 1e3),
         "* clocks: %s" % json.dumps(b.get("clocks")),
         "* cpu_baseline (C oracle, %d threads): %.3e agent-env-steps/s" % (b["cpu_baseline"]["cores"], b["cpu_baseline"]["value"])]
for name, f in [("c3", "bench_c3.json"), ("c4 (COVID)", "bench_c4.json"), ("c5", "bench_c5.json")]:
    p = os.path.join(OUT, f)
    if os.path.exists(p):
        d = json.load(open(p))
        lines.append("* %s: %.3e agent-env-steps/s, %.4f ms/step, dominant-kernel frac %.3f"
                     % (name, d["value"], d["ms_per_step"], d["roofline"]["frac"]))
if shares:
    lines += ["", "## ncu launch list (`--metrics gpu__time_duration.sum --clock-control none`, cold-cache, serialised)", "",
              "| kernel | launches | avg us | share |", "|---|---|---|---|"]
    lines += ["| %s | %d | %.1f | %.1f%% |" % s for s in sorted(shares, key=lambda s: -s[3])]
if "aie_step_kernel" in raw:
    d, u, _ = raw["aie_step_kernel"]
    lines += ["", "## ncu --set full, fused step kernel, one launch (%s_ncu_full_aie_step_kernel_raw.csv)" % tag, ""]
    for kk in ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread",
               "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "launch__waves_per_multiprocessor",
               "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
               "smsp__issue_active.avg.pct_of_peak_sustained_active", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
               "sm__icc_request_hit_rate.pct", "smsp__thread_inst_executed_per_inst_executed.ratio"]:
        lines.append("* %s = %s %s" % (kk, d.get(kk), u.get(kk, "")))
    stall = {kk.split("stalled_")[1].replace("_per_issue_active.ratio", ""): float(v) for kk, v in d.items()
             if "issue_stalled" in kk and kk.endswith("per_issue_active.ratio") and "not_issued" not in kk}
    lines.append("")
    lines.append("warp stall reasons (warp-cycles per issued instruction): " +
                 ", ".join("%s %.2f" % kv for kv in sorted(stall.items(), key=lambda x: -x[1])[:10]))
    tr = float(d["dram__bytes_read.sum"]) + float(d["dram__bytes_write.sum"])
    lines.append("")
    lines.append("traffic = dram read + write = %.1f MB per launch vs %.1f MB algorithmic: no re-reads; the L2 (50 MB) absorbs part "
                 "of the record write-back." % (tr, k["aie_step_kernel"]["alg_bytes_per_launch"] / 1e6))
for f in ("racecheck.log", "memcheck.log"):
    p = os.path.join(OUT, f)
    if os.path.exists(p):
        tail = [l for l in open(p).read().splitlines() if "SUMMARY" in l]
        lines.append("* %s: %s" % (f, tail[-1].strip("= ") if tail else "?"))
open(os.path.join(PROF, "%s_SUMMARY.md" % tag), "w").write("\n".join(lines) + "\n")
print("\n".join(lines))
