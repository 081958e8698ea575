#!/bin/bash
# Zillow `value` (device-resident, lanes overlapping) under scheduling knobs; one line per variant -> gpurun_out/bench_variants.log
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
run() { echo "== $*"; env "$@" python bench.py --workload zillow --steps 10 --no-cpu-baseline --no-pageable 2>/dev/null | python -c "
import json,sys
d=json.loads(sys.stdin.read().strip().splitlines()[-1])
print('value %.2f G rows/s  ms/step %.3f  roofline %.3f  e2e %.3f G rows/s  kernel_ms/launch %.3f' % (d['value']/1e9, d['ms_per_step'], d['roofline']['frac'], d['e2e']['value']/1e9, d['roofline']['kernel_ms_per_launch']))"; }
{
run TPLX_LANES=2
run TPLX_LANES=1
run TPLX_LANES=3
run TPLX_LANES=2 TPLX_MASK_OCC=3
run TPLX_LANES=3 TPLX_MASK_OCC=3
run TPLX_LANES=2 TPLX_MASK_OCC=2
} 2>&1 | tee gpurun_out/bench_variants.log
