#!/bin/bash
# A/B of library build variants on one GPU: tools/ab_run.sh <out-dir> <tag> <variant> [<variant> ...]   ("base" = product build)
out=$1; tag=$2; shift 2
mkdir -p "$out"
for v in "$@"; do
  if [ "$v" = "base" ]; then unset SPB_LIB_PATH; else export SPB_LIB_PATH=$PWD/spectre_b200/libspectre_b200_$v.so; fi
  echo "=== variant $v" >> "$out/${tag}_ab.log"
  python tools/microbench.py modmul_quick >> "$out/${tag}_ab.log" 2>&1
  python bench.py --steps 40 --warmup 5 --no-prove --no-cpu-baseline >> "$out/${tag}_ab.log" 2>&1
done
