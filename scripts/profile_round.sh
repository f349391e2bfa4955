#!/bin/bash
# One GPU-box call that produces everything profiles/ holds for a round (run under gpurun, 1 GPU):
#   gpurun --timeout 2400 -- 'bash scripts/profile_round.sh r02'
# Numbers printed by the runs under ncu are never bench values; the bench JSON comes from the plain runs.
R=${1:-r02}
O=gpurun_out
mkdir -p $O
set -x
timeout 900 python -m pytest tests -m gpu -q > $O/${R}_pytest_gpu.log 2>&1; echo "pytest rc=$?" >> $O/${R}_pytest_gpu.log
timeout 600 python bench.py > $O/${R}_bench_1gpu.json 2> $O/${R}_bench_1gpu.err; echo "bench rc=$?"
for w in fanout mixed reply; do
  timeout 600 python bench.py --workload $w > $O/${R}_bench_$w.json 2> $O/${R}_bench_$w.err; echo "$w rc=$?"
done
timeout 600 python bench.py --impl reference --steps 3 --warmup 1 > $O/${R}_bench_reference.json 2> $O/${R}_bench_reference.err; echo "reference rc=$?"
# launch list of the same bench command (per-launch times are cold-cache and serialised: compare shares, not absolutes)
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 800 --csv --log-file $O/${R}_launches.csv \
    python bench.py --steps 2 --warmup 3 --events 262144 --cpu-sample 2000 > $O/${R}_launches_bench.log 2>&1
# full captures of the heaviest kernels (one launch each, after warm-up launches)
for k in walk plan_tool emit; do
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:ck_${k}_kernel -s 3 -c 1 -f -o $O/${R}_${k} \
      python scripts/quick_bench.py 1048576 > $O/${R}_ncu_${k}.log 2>&1
done
timeout 900 ncu --set full --clock-control none --import-source on -k regex:ck_walk_long_kernel -s 2 -c 1 -f -o $O/${R}_walk_long \
    python scripts/quick_fanout.py 4096 > $O/${R}_ncu_walk_long.log 2>&1
# the long-record decode of the mixed workload: warp pre-scan and one thread per history message
timeout 900 ncu --set full --clock-control none --import-source on -k regex:ck_walk_long_kernel -s 2 -c 1 -f -o $O/${R}_prescan_mixed \
    python scripts/quick_mixed.py 65536 > $O/${R}_ncu_prescan_mixed.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:ck_walk_elems_kernel -s 2 -c 1 -f -o $O/${R}_walk_elems \
    python scripts/quick_mixed.py 65536 > $O/${R}_ncu_walk_elems.log 2>&1
# summaries are made here (ncu is on the box); the reports themselves are too large to bring back
PROFILES_OUT=$O/profiles_$R KEEP_REP=0 python scripts/make_profiles.py $R > $O/${R}_make_profiles.log 2>&1
rm -f $O/*.ncu-rep
cuobjdump -sass calfkit-sdk_b200/libcalfkit_b200.so | grep -E "LDGSTS|UBLKCP|SYNCS|ATOM|RED\." | awk '{print $2}' | sort | uniq -c | sort -rn | head -20 > $O/${R}_sass_mnemonics.txt
ls -la $O
