"""K9 merge of resolved rows at block size: one 16 M-row stage result with i64, str and Option[i64] outputs and 1 % exception rows,
90 % of them resolved, then tplx_gpu_result_merge_resolved timed with a host clock (the call ends in a synchronise):
  python tools/merge_probe.py            # prints the median of 7 merges after one warm-up, and the merge's kernel ms"""
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tuplex_b200 import backend, frontend  # noqa: E402
from tuplex_b200.backend import Column, pack_valid  # noqa: E402
from tuplex_b200.ir import T_I64, T_STR  # noqa: E402

n = int(os.environ.get("MERGE_ROWS", str(16 << 20)))
rng = np.random.default_rng(7)


def strs(m):  # m strings of 8 lowercase letters
    return Column(T_STR, rng.integers(97, 123, m * 8).astype(np.uint8), (np.arange(m + 1, dtype=np.uint64) * 8).astype(np.uint32))


k = rng.integers(1, 1000, n).astype(np.int64)
k[rng.random(n) < 0.01] = 0  # ZeroDivisionError
cols = [Column(T_I64, k), strs(n), Column(T_I64, rng.integers(0, 1 << 40, n), None, pack_valid(rng.random(n) >= 0.1))]
sc = frontend.StageCompiler([T_I64, T_STR, T_I64], ["k", "s", "o"], [2])
sc.add_map(lambda x: (100 // x["k"], x["s"], x["o"]), 100001)
backend.init([0])
st = backend.Stage(sc.finish_memory())
blk = backend.Block.upload(0, cols, n)
res = st.run(blk)
exc = np.sort(res.exceptions()["row_no"])
res_nos = np.sort(rng.choice(exc, int(len(exc) * 0.9), replace=False))
m = len(res_nos)
rblk = backend.Block.upload(0, [Column(T_I64, rng.integers(-5, 5, m)), strs(m),
                                Column(T_I64, rng.integers(0, 1 << 40, m), None, pack_valid(rng.random(m) >= 0.1))], m)
print("stage: %d rows -> %d normal rows, %d exceptions, %d resolved" % (n, int(res.info.n_out_rows), len(exc), m))
times, kms = [], []
for it in range(8):
    t0 = time.perf_counter()
    merged = res.merge_resolved(rblk, res_nos.tolist())
    dt = (time.perf_counter() - t0) * 1e3
    info = merged.info
    if it:  # the first call is the warm-up
        times.append(dt)
        kms.append(info.kernel_ms)
    launches, n_out = int(info.kernel_launches), int(info.n_out_rows)
    merged.free()
print("merge_resolved: %d out rows, %d launches, wall median %.3f ms (min %.3f, max %.3f), kernel median %.3f ms over %d calls"
      % (n_out, launches, statistics.median(times), min(times), max(times), statistics.median(kms), len(times)))
rblk.free()
res.free()
blk.free()
st.close()
