"""Turns what scripts/profile_round.sh left in gpurun_out/ into the tracked summaries under profiles/ (run here, no GPU):
   python scripts/make_profiles.py r01 [n_records_of_the_ncu_runs=1048576]"""
import csv, json, os, shutil, subprocess, sys
R = sys.argv[1] if len(sys.argv) > 1 else "r02"
NREC = int(sys.argv[2]) if len(sys.argv) > 2 else 1048576
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G, P = os.path.join(ROOT, "gpurun_out"), os.environ.get("PROFILES_OUT") or os.path.join(ROOT, "profiles")
KEEP_REP = os.environ.get("KEEP_REP", "1") == "1"       # on the GPU box: summaries only (the reports exceed what gpurun brings back)
os.makedirs(P, exist_ok=True)
for name in ("bench_1gpu", "bench_fanout", "bench_mixed", "bench_reply", "bench_reference", "bench_2gpu", "bench_4gpu", "bench_8gpu"):
    src = os.path.join(G, f"{R}_{name}.json")
    if os.path.exists(src):
        lines = [l for l in open(src).read().splitlines() if l.startswith("{")]
        if lines:
            open(os.path.join(P, f"{R}_{name}.json"), "w").write(lines[-1] + "\n")
for name in ("launches.csv", "pytest_gpu.log", "sass_mnemonics.txt", "exchange_parity_2gpu.log"):
    src = os.path.join(G, f"{R}_{name}")
    if os.path.exists(src):
        shutil.copy(src, os.path.join(P, f"{R}_{name}"))
traffic = {}
def nrec_of(k): return 4096 if k == "walk_long" else (65536 if k in ("prescan_mixed", "walk_elems") else NREC)
for k, short in (("walk", "walk"), ("plan_tool", "plan"), ("emit", "emit"), ("walk_long", "walk_long"), ("prescan_mixed", "prescan_mixed"), ("walk_elems", "walk_elems")):
    rep = os.path.join(G, f"{R}_{k}.ncu-rep")
    if not os.path.exists(rep):
        continue
    if KEEP_REP: shutil.copy(rep, os.path.join(P, f"{R}_{k}.ncu-rep"))
    s1 = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "ncu_summary.py"), rep], capture_output=True, text=True).stdout
    s2 = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "ncu_lines.py"), rep, "25"], capture_output=True, text=True).stdout
    open(os.path.join(P, f"{R}_{k}.txt"), "w").write(
        f"ncu --set full --clock-control none --import-source on, one launch of the kernel over {nrec_of(k)} records (scripts/profile_round.sh)\n"
        "numbers under a profiler are not bench values\n\n" + s1 + "\n" + s2)
    rows = list(csv.reader(subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout.splitlines()))
    hdr, unit, val = rows[0], rows[1], rows[2]
    def metric(name):
        i = hdr.index(name); v = float(val[i]); u = unit[i].lower()
        return v * {"gbyte": 1e9, "mbyte": 1e6, "kbyte": 1e3, "byte": 1.0}.get(u, 1.0)
    nrec = 4096 if k == "walk_long" else (65536 if k in ("prescan_mixed", "walk_elems") else NREC)
    traffic[short] = {"dram_bytes_per_record": (metric("dram__bytes_read.sum") + metric("dram__bytes_write.sum")) / nrec,
                      "source": f"profiles/{R}_{k}.ncu-rep (dram__bytes_read.sum + dram__bytes_write.sum) / {nrec} records"}
if traffic:
    json.dump(traffic, open(os.path.join(P, "traffic.json"), "w"), indent=1)
# kernel shares of a step from the launch list (cold-cache, serialised: compare shares, not absolutes)
lp = os.path.join(G, f"{R}_launches.csv")
if os.path.exists(lp):
    tot = {}
    rows = [r for r in csv.reader(open(lp)) if len(r) > 5]
    hdr = next((r for r in rows if "Kernel Name" in r), None)
    if hdr:
        ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
        for r in rows:
            if r is hdr or len(r) <= vi: continue
            try: v = float(r[vi].replace(",", ""))
            except ValueError: continue
            name = r[ki].split("(")[0]
            tot[name] = tot.get(name, [0.0, 0]); tot[name][0] += v; tot[name][1] += 1
        s = sum(v[0] for v in tot.values())
        with open(os.path.join(P, f"{R}_launches_summary.txt"), "w") as f:
            f.write("ncu --metrics gpu__time_duration.sum --clock-control none over `bench.py --steps 2 --warmup 3 --events 262144`\n"
                    "per-launch times are cold-cache and serialised: shares, not absolutes\n\n")
            for k, v in sorted(tot.items(), key=lambda kv: -kv[1][0]):
                f.write(f"{100 * v[0] / s:6.2f} %  {v[0] / 1e3:10.1f} us total  {v[1]:4d} launches  {k}\n")
print(open(os.path.join(P, "traffic.json")).read() if traffic else "no ncu reps")
