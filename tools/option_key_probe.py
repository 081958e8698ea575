"""aggregateByKey over an Option[str] key: the bench's aggregateByKey shape (125 M rows, 10 M distinct string keys, i64 sum) with
10 % of the keys None, next to the same data with no validity bitmap, the plain (non-Option) stage, and the plain stage with the same
10 % of the rows on one ordinary key (a hot group without None). Prints rows/s per variant from
host-clock timings of stage runs that end in a device synchronise (K4's run reads its counters back), plus the CUDA-event kernel time:
  python tools/option_key_probe.py          # ROWS=..., KEYS=..., REPEAT=... override the shape"""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tuplex_b200 import backend, frontend, workloads  # noqa: E402
from tuplex_b200.ir import T_I64, T_STR  # noqa: E402

n, n_keys = int(os.environ.get("ROWS", "125000000")), int(os.environ.get("KEYS", "10000000"))
repeat = int(os.environ.get("REPEAT", "5"))
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
key, val = workloads.gen_keyed(n, n_keys, seed=42)
none = np.random.default_rng(7).random(n) < 0.1
option_key = backend.Column(T_STR, key.data, key.offsets, backend.pack_valid(~none))
# the same 10 % of the rows on one ordinary key instead of None: one hot group with no Option key involved
hot = key.data.reshape(-1, 8).copy()
hot[none] = np.frombuffer(b"hotgroup", np.uint8)
hot_key = backend.Column(T_STR, hot.reshape(-1), key.offsets)


def stage(option: bool):
    sc = frontend.StageCompiler([T_STR, T_I64], ["key", "v"], option_cols=[0] if option else ())
    return backend.Stage(sc.finish_hash(["key"], lambda a, x: a + x[1], lambda a, b: a + b, 0, 100001))


backend.init([0])
variants = [("plain stage, no Option key", stage(False), key), ("plain stage, 10% on one key", stage(False), hot_key),
            ("Option key, no bitmap", stage(True), key), ("Option key, 10% None", stage(True), option_key)]
for name, st, kcol in variants:
    blk = backend.Block.upload(0, [kcol, val], n)
    walls, kernels = [], []
    for r in range(repeat + 1):
        st.hash_reset(0)
        st.hash_reserve(0, n_keys)
        t0 = time.perf_counter()
        res = st.run(blk)
        info = res.info
        t1 = time.perf_counter()
        if r:  # the first run warms up
            walls.append(t1 - t0)
            kernels.append(info.kernel_ms)
        res.free()
    fin = st.hash_finish(0)
    groups = int(fin.info.n_out_rows)
    fin.free()
    blk.free()
    w, k = float(np.median(walls)), float(np.median(kernels))
    print("%-28s groups %9d  run %.2f ms (%.3f G rows/s)  K4 kernel %.2f ms (%.3f G rows/s)" % (name, groups, w * 1e3, n / w / 1e9, k, n / k / 1e6))
