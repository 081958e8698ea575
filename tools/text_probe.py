"""What K10 (the device text source, tplx_gpu_text_parse) costs, and what it saves Context.text, on the reference's Apache logs.

The logs fixture (tests/golden/logs.sample.txt.gz) is replicated to about 1 GB; a seeded variant has CRLF line ends and 1 % of
its lines made invalid UTF-8 (a 0xFF byte). For each file, in one process:
  * upload_ms: tplx_gpu_csv_upload of the whole file, host clock ending in a device synchronise;
  * parse_ms: K10's CUDA-event time, median of 7 runs after 2 warm-ups, with its algorithmic bytes (input read 3x, the column
    written once, line ends + per-line scratch + offsets + rowmap) and the rate they give;
  * the logs pipeline with a small output (ParseWithStrip, then unique of `method`) through Context, host clock around
    text() + collect() (collect returns host rows, so it ends after the device has finished), over K10 and over the host
    reader (read_lines + parallelize, the path Context.text took before K10), alternating, 3 runs each.
Prints one JSON object; with --out it is also written to that file.

    python tools/text_probe.py [--mb 1000] [--out results.json]
"""
import argparse
import gzip
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tuplex_b200  # noqa: E402
from tuplex_b200 import backend  # noqa: E402
from tuplex_b200.textsource import read_lines  # noqa: E402
from logs_udfs import ParseWithStrip  # noqa: E402


def make_files(dirname: str, mb: int):
    sample = gzip.open(os.path.join(ROOT, "tests", "golden", "logs.sample.txt.gz"), "rb").read()
    reps = max(1, mb * 1000 * 1000 // len(sample))
    plain = os.path.join(dirname, "logs.txt")
    with open(plain, "wb") as f:
        for _ in range(reps):
            f.write(sample)
    rng = random.Random(2026)
    lines = sample.split(b"\n")
    for i in rng.sample(range(len(lines) - 1), (len(lines) - 1) // 100):
        k = rng.randrange(len(lines[i]) + 1)
        lines[i] = lines[i][:k] + b"\xff" + lines[i][k:]
    variant = b"\r\n".join(lines)
    crlf = os.path.join(dirname, "logs_crlf_invalid.txt")
    reps_v = max(1, mb * 1000 * 1000 // len(variant))
    with open(crlf, "wb") as f:
        for _ in range(reps_v):
            f.write(variant)
    return plain, crlf


def sync():
    import torch
    torch.cuda.synchronize(0)


def k10(path: str):
    import numpy as np
    data = np.fromfile(path, dtype=np.uint8)
    sync()
    t0 = time.perf_counter()
    buf = backend.CsvBuffer(0, data)
    sync()
    upload_ms = (time.perf_counter() - t0) * 1e3
    times, info = [], None
    for k in range(9):
        p = buf.parse_text()
        info = p.info
        out_bytes = p.block_bytes()[0]
        if k >= 2:
            times.append(float(info.parse_ms))
        p.free()
    buf.free()
    n, nl = int(data.size), int(info.n_rows)
    alg = 3 * n + out_bytes + nl * (4 + 17 + 8)
    med = statistics.median(times)
    return {"bytes": n, "lines": nl, "upload_ms": upload_ms, "parse_ms_median": med, "parse_ms_all": times,
            "algorithmic_bytes": alg, "algorithmic_GBps": alg / med / 1e6, "kernel_launches": int(info.kernel_launches)}


def pipeline(ds):
    return ds.map(ParseWithStrip).map(lambda x: x["method"]).unique().collect()


def run_device(path):
    ctx = tuplex_b200.Context()
    t0 = time.perf_counter()
    rows = pipeline(ctx.text(path))
    dt = time.perf_counter() - t0
    assert ctx.metrics.text_rows > 0 and not any("falls back" in m for m in ctx._messages), ctx._messages
    return dt, rows, ctx.metrics.text_parse_ms


def run_host(path):
    ctx = tuplex_b200.Context()
    t0 = time.perf_counter()
    rows = pipeline(ctx.parallelize(read_lines([path], print)))
    return time.perf_counter() - t0, rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=1000)
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    args = ap.parse_args()
    backend.init([0])
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": q.stdout.strip()}
    with tempfile.TemporaryDirectory() as td:
        for name, path in zip(("logs", "logs_crlf_1pct_invalid"), make_files(td, args.mb)):
            r = k10(path)
            print(name, "K10", json.dumps(r), flush=True)
            dev_s, host_s = [], []
            for _ in range(3):
                dt, rows_d, parse_ms = run_device(path)
                dev_s.append(dt)
                ht, rows_h = run_host(path)
                host_s.append(ht)
                assert rows_d == rows_h, (rows_d, rows_h)
                print(name, "pipeline device %.3f s, host reader %.3f s" % (dt, ht), flush=True)
            r.update({"pipeline_device_s": dev_s, "pipeline_host_reader_s": host_s, "pipeline_text_parse_ms": parse_ms,
                      "pipeline_rows": len(rows_d)})
            out[name] = r
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
