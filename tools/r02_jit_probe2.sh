#!/bin/bash
# specialiser experiments: K1v occupancy / pipelined loop, dense-launch prefetch, specialised mask kernel vs closed form
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
timeout 600 python -m pytest tests/test_jit.py -x -q 2>&1 | tail -5
for mb in 6 8; do echo "== C1 JIT minb $mb"; TPLX_JIT_MINB_VEC=$mb timeout 120 python tools/c1_probe.py 2>&1 | tail -1; done
for mb in 4 5 6; do echo "== C1 JIT PIPE minb $mb"; TPLX_JIT_VEC_PIPE=1 TPLX_JIT_MINB_VEC=$mb timeout 120 python tools/c1_probe.py 2>&1 | tail -1; done
echo "== C1 JIT PIPE parity"; TPLX_JIT_VEC_PIPE=1 timeout 300 python -m pytest tests/test_jit.py -x -q -k "c1_specialised or fixed_width" 2>&1 | tail -3
echo "== zillow JIT default"; timeout 120 python tools/kernel_probe.py 2>&1 | tail -3
echo "== zillow JIT no prefetch"; TPLX_JIT_PREFETCH=0 timeout 120 python tools/kernel_probe.py 2>&1 | tail -3
echo "== zillow JIT minb 2"; TPLX_JIT_MINB=2 timeout 120 python tools/kernel_probe.py 2>&1 | tail -3
echo "== zillow JIT minb 4"; TPLX_JIT_MINB=4 timeout 120 python tools/kernel_probe.py 2>&1 | tail -3
for mb in 3 4 5; do echo "== zillow JIT mask (instead of K1f) minb $mb"; TPLX_JIT_MASK=1 TPLX_JIT_MINB_MASK=$mb timeout 120 python tools/kernel_probe.py 2>&1 | tail -3; done
echo "== zillow JIT mask parity"; TPLX_JIT_MASK=1 TPLX_JIT=2 timeout 300 python -m pytest tests/test_jit.py tests/test_gpu_parity.py -x -q -k "zillow or prefilter" 2>&1 | tail -3
echo "== q6 through the specialised K3 (no fused hint)"; TPLX_NO_FUSED=1 timeout 200 python bench.py --workload q6 --rows 200000000 --steps 3 --warmup 2 --no-cpu-baseline --no-pageable 2>&1 | python -c "import sys,json; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print(d['value'], d['roofline'])"
echo "== q6 interpreted K3 (no fused hint)"; TPLX_JIT=0 TPLX_NO_FUSED=1 timeout 200 python bench.py --workload q6 --rows 200000000 --steps 3 --warmup 2 --no-cpu-baseline --no-pageable 2>&1 | python -c "import sys,json; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print(d['value'], d['roofline'])"
echo "== ncu: specialised K1v on C1 (50M rows)"
PROBE_ROWS=50000000 timeout 300 ncu --set full --clock-control none --import-source on -k regex:tplx_jit_kernel -s 2 -c 1 -f -o gpurun_out/r02_jit_vec python tools/c1_probe.py > gpurun_out/ncu_jv.log 2>&1; tail -2 gpurun_out/ncu_jv.log
echo "== ncu: specialised dense launch (Zillow)"
timeout 300 ncu --set full --clock-control none --import-source on -k regex:tplx_jit_kernel -s 3 -c 1 -f -o gpurun_out/r02_jit_dense python tools/kernel_probe.py > gpurun_out/ncu_jd.log 2>&1; tail -2 gpurun_out/ncu_jd.log
