"""Zillow Z1 kernel split: the prefilter (K1f plus the mask count / scan / expand kernels) and the dense K1 launch over its
survivors, over one device-resident block of 16,330,500 rows (500 cycles of the fixture, the block size bench.py uses).

Prints the card and its power limit, then the median CUDA-event time of each interval over REPEAT runs after WARMUP runs, the
rows kernel's launch shape (tile rows per thread, shared memory, CTAs per SM):
  python tools/dense_probe.py            # CYCLES=..., REPEAT=..., WARMUP=... override the shape; TPLX_GPU_LIB picks the library
"""
import os
import re
import subprocess
import sys
import tempfile

os.environ.setdefault("TPLX_JIT_SYNC", "1")  # steady state: the specialised kernels from the first run on
os.environ["TPLX_TRACE"] = "1"  # the library prints each interval of result_info and the rows kernel's launch shape on stderr

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tuplex_b200 import backend, workloads as W  # noqa: E402

cycles = int(os.environ.get("CYCLES", "500"))
repeat = int(os.environ.get("REPEAT", "12"))
warmup = int(os.environ.get("WARMUP", "3"))
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()

backend.init([0])
src, n0 = W.load_zillow_fixture()
n = cycles * n0
cols = W.replicate(src, n0, n)
st = backend.Stage(W.zillow_program())
blk = backend.Block.upload(0, cols, n)

# the trace goes to fd 2 from native code: send it to a file for the timed runs
log = tempfile.TemporaryFile(mode="w+b")
saved = os.dup(2)
os.dup2(log.fileno(), 2)
out_rows = 0
try:
    for it in range(warmup + repeat):
        r = st.run(blk)
        inf = r.info
        out_rows = int(inf.n_out_rows)
        r.free()
        sys.stderr.flush()
        os.write(2, b"[probe] end of run\n")
finally:
    os.dup2(saved, 2)
    os.close(saved)
log.seek(0)
text = log.read().decode(errors="replace")
runs = text.split("[probe] end of run\n")[:-1][warmup:]
dense, pre, shape = [], [], ""
for chunk in runs:
    m = re.search(r"stage kernels ([0-9.]+) ms", chunk)
    p = re.findall(r"prefilter ([0-9.]+) ms", chunk)
    s = re.findall(r"rows kernel[^\n]*", chunk)
    if m:
        dense.append(float(m.group(1)))
    if p:
        pre.append(sum(float(x) for x in p))
    if s:
        shape = s[-1]
lib = os.environ.get("TPLX_GPU_LIB", "tuplex_b200/lib/libtplx_gpu.so")
print(f"card: {card}")
print(f"library: {lib}; rows {n}, survivors written {out_rows}")
print(f"  {shape}")
if dense and pre:
    print(f"  prefilter (K1f + mask kernels): median {np.median(pre) * 1e3:.0f} us  [min {min(pre) * 1e3:.0f}, max {max(pre) * 1e3:.0f}] over {len(pre)} runs")
    print(f"  dense K1 over the survivors:    median {np.median(dense) * 1e3:.0f} us  [min {min(dense) * 1e3:.0f}, max {max(dense) * 1e3:.0f}]")
else:
    print("  no interval found in the trace")
blk.free()
