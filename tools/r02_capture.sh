#!/bin/bash
# Round-2 evidence in ONE gpurun call: GPU tests, the default bench line (+ reference arm), the ncu launch list of the same
# command and one `ncu --set full` capture of each flagship kernel. Everything lands in gpurun_out/r02_*.
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
O=gpurun_out
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm --format=csv > $O/r02_gpu.txt 2>&1
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > $O/r02_smoke.log 2>&1; echo "smoke rc=$?" >> $O/r02_smoke.log; tail -2 $O/r02_smoke.log
if [ -n "${QUICK_TESTS:-}" ]; then
  timeout 300 python -m pytest $QUICK_TESTS -m gpu -q > $O/r02_pytest_quick.log 2>&1; echo "pytest rc=$?" >> $O/r02_pytest_quick.log; tail -3 $O/r02_pytest_quick.log
fi
if [ "${SKIP_TESTS:-0}" != "1" ]; then
  timeout 900 python -m pytest tests -m gpu -q > $O/r02_pytest_gpu.log 2>&1; echo "pytest rc=$?" >> $O/r02_pytest_gpu.log
  tail -3 $O/r02_pytest_gpu.log
fi
timeout 600 python bench.py --impl reference --steps 3 --warmup 1 > $O/r02_bench_reference_arm.json 2> $O/r02_bench_reference_arm.err
timeout 900 python bench.py > $O/r02_bench_default.json 2> $O/r02_bench_default.err; echo "bench rc=$?"
tail -c 600 $O/r02_bench_default.json
# launch list of the same command (short: 2 steps, no CPU arms); per-launch times are serialised / cold-cache
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file $O/r02_launches.csv \
  python bench.py --steps 2 --warmup 1 --no-cpu-baseline --no-pageable --no-extras > $O/r02_launches_bench.log 2>&1
# one full capture per flagship kernel
export PROBE_CYCLES=${PROBE_CYCLES:-400}
[ "${SKIP_OLD:-0}" = "1" ] || timeout 300 ncu --set full --clock-control none --import-source on -k regex:stage_mask -s 3 -c 1 -f -o $O/r02_scan python tools/kernel_probe.py > $O/ncu_a.log 2>&1
# the dense launch and the C1 kernel are the stage specialiser's builds (tplx_jit_kernel) by default; TPLX_JIT=0 = their interpreting twins
timeout 300 ncu --set full --clock-control none --import-source on -k regex:tplx_jit_kernel -s 3 -c 1 -f -o $O/r02_dense python tools/kernel_probe.py > $O/ncu_b.log 2>&1
PROBE_ROWS=50000000 timeout 300 ncu --set full --clock-control none --import-source on -k regex:tplx_jit_kernel -s 2 -c 1 -f -o $O/r02_vec python tools/c1_probe.py > $O/ncu_c.log 2>&1
ls -la $O/*.ncu-rep
# K8: every kernel of one probe of the bench's join workload (count, scan, emit, gathers)
timeout 200 python tools/join_probe.py > $O/r02_join_probe.log 2>&1
PROBE_REPEAT=1 timeout 300 ncu --set full --clock-control none --import-source on -k regex:join_ -c 14 -f -o $O/r02_join python tools/join_probe.py > $O/ncu_e.log 2>&1
[ "${SKIP_OLD:-0}" = "1" ] || timeout 300 ncu --set full --clock-control none --import-source on -k regex:fused_scan_agg_tma -s 1 -c 1 -f -o $O/r02_q6 python bench.py --workload q6 --rows 100000000 --steps 1 --warmup 1 --no-cpu-baseline --no-pageable > $O/ncu_d.log 2>&1
ls -la $O/*.ncu-rep
