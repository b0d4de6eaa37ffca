#!/bin/bash
# A/B harness for kernel experiments (one GPU): builds of the library with different -D switches
# live in variants/lib_<name>.so (scratch, git-ignored) and are selected through SLB_LIBRARY; prints the per-kernel breakdown of
# one step for each.  Usage: bash profiles/run_variants.sh base name1 name2 ...
for lib in "$@"; do
  if [ $lib = base ]; then unset SLB_LIBRARY; else export SLB_LIBRARY="$(cd "$(dirname "$0")/.." && pwd)/variants/lib_$lib.so"; fi
  timeout 200 python bench.py --no-cpu-baseline --no-e2e --steps 100 --warmup 10 2>/dev/null | python -c "
import sys, json
d = json.loads(sys.stdin.read().strip().splitlines()[-1])
print('$lib', 'ms/step %.4f' % d['ms_per_step'], {k: round(v * 1e3, 1) for k, v in d['roofline']['kernel_ms'].items()})"
done
