"""DataSet.cache() on the device against the host cache (the rows through CPython and a new host source, which is what cache()
did before and still does where the device cache is not taken). Prints one JSON object; --out also writes it to a file.

  zillow   Z1 in the reference's --preload form: ctx.csv(fixture replicated k times).cache(), then Z1 and tocsv; cache time,
           post-cache pipeline time and the output's md5, device and host cache alternating (--zillow-host-copies), then the
           device cache alone at --zillow-copies
  logs     runtuplex-io's shape: ctx.text(logs).cache() and ctx.csv(blacklist).cache(), then the parse and the join, on the logs
           sample replicated to about --logs-mb MB (device cache only; the host cache at --logs-host-mb)
  bytes    ctx.metrics.cache_bytes of each cache against the exact column bytes (values, string bytes + offsets, bitmaps)
"""
import argparse
import gzip
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tuplex_b200  # noqa: E402
from tuplex_b200 import dataset, workloads  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _cache(ds, mode):
    if mode == "device":
        return ds.cache()
    rows, names = ds._execute()  # the host cache
    return ds._ctx._dataset_from_rows(rows, names)


def _exact_bytes(src):
    tot = 0
    for p in src.rows.parts:
        n = int(p.info.n_out_rows)
        for c, t in enumerate(src.col_types):
            tot += (int(p.info.out_str_bytes[c]) + (n + 1) * 4) if t == workloads.T_STR else n * 8
            tot += (n + 31) // 32 * 4 if c in src.option_cols else 0
    return tot


def zillow(tmp, k, mode):
    data = gzip.open(os.path.join(workloads.GOLDEN, "zillow_noexc.csv.gz"), "rb").read()
    head, body = data.split(b"\n", 1)
    path = os.path.join(tmp, "zillow_%d.csv" % k)
    if not os.path.exists(path):
        with open(path, "wb") as fp:
            fp.write(head + b"\n" + body * k)
    ctx = tuplex_b200.Context()
    t0 = time.perf_counter()
    ds = _cache(ctx.csv(path), mode)
    t1 = time.perf_counter()
    out = os.path.join(tmp, "z_out_%s_%d" % (mode, k))
    workloads.zillow_pipeline(ds).tocsv(out)
    t2 = time.perf_counter()
    md5 = hashlib.md5(open(os.path.join(out, "part0.csv"), "rb").read()).hexdigest()
    r = {"mode": mode, "copies": k, "rows": 32661 * k, "cache_s": round(t1 - t0, 3), "pipeline_s": round(t2 - t1, 3), "md5": md5,
         "cache_rows": ctx.metrics.cache_rows}
    if isinstance(ds._source, dataset.CacheSource):
        r.update(cache_bytes=ctx.metrics.cache_bytes, exact_bytes=_exact_bytes(ds._source))
    return r


def logs(tmp, mb, mode):
    from logs_udfs import ParseWithStrip
    sample = gzip.open(os.path.join(ROOT, "tests", "golden", "logs.sample.txt.gz"), "rb").read()
    k = max(1, int(mb * 1e6) // len(sample))
    path = os.path.join(tmp, "logs_%d.txt" % k)
    if not os.path.exists(path):
        with open(path, "wb") as fp:
            fp.write(sample * k)
    ips = os.path.join(tmp, "ip_blacklist.csv")
    with open(ips, "wb") as fp:
        fp.write(gzip.open(os.path.join(ROOT, "tests", "golden", "ip_blacklist.csv.gz"), "rb").read())
    ctx = tuplex_b200.Context()
    t0 = time.perf_counter()
    text, bad = _cache(ctx.text(path), mode), _cache(ctx.csv(ips), mode)
    t1 = time.perf_counter()
    out = os.path.join(tmp, "l_out_%s_%d" % (mode, k))
    text.map(ParseWithStrip).join(bad, "ip", "BadIPs").selectColumns(["ip", "endpoint"]).tocsv(out)
    t2 = time.perf_counter()
    md5 = hashlib.md5(open(os.path.join(out, "part0.csv"), "rb").read()).hexdigest()
    r = {"mode": mode, "bytes": len(sample) * k, "cache_s": round(t1 - t0, 3), "pipeline_s": round(t2 - t1, 3), "md5": md5,
         "cache_rows": ctx.metrics.cache_rows}
    if isinstance(text._source, dataset.CacheSource):
        r.update(cache_bytes=ctx.metrics.cache_bytes, exact_bytes=_exact_bytes(text._source) + _exact_bytes(bad._source))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--zillow-host-copies", type=int, default=20)
    ap.add_argument("--zillow-copies", type=int, default=400)
    ap.add_argument("--logs-mb", type=float, default=1000)
    ap.add_argument("--logs-host-mb", type=float, default=20)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": _card(), "zillow": [], "logs": []}
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(a.repeats):
            for mode in ("device", "host"):
                res["zillow"].append(zillow(tmp, a.zillow_host_copies, mode))
                res["logs"].append(logs(tmp, a.logs_host_mb, mode))
        res["zillow"].append(zillow(tmp, a.zillow_copies, "device"))
        res["logs"].append(logs(tmp, a.logs_mb, "device"))
    txt = json.dumps(res)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt + "\n")


if __name__ == "__main__":
    main()
