#!/bin/bash
# A/B timing of alternative builds of the library (gpurun_variants/*.so, git-ignored) against the in-tree one.
N=${1:-1048576}
echo "== default"; python scripts/quick_bench.py $N 2>&1 | grep -E "walk|plan|emit|pipelined|status"
for so in gpurun_variants/*.so; do
  echo "== $so"; CK_LIB=$PWD/$so python scripts/quick_bench.py $N 2>&1 | grep -E "walk|plan|emit|pipelined|status"
done
