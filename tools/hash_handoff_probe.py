"""What the device key sort (K11) costs, and what aggregateByKey / unique() pipelines cost end to end now that their groups stay on
the device.

  * sort: tplx_gpu_result_sort_by_keys alone over --rows rows of a stage result: i64 keys (uniform over all 64 bits), string keys of
    the aggbykey shape but 8-16 bytes long ('k' + 7 digits + 0-8 letters), and a two-column key (that string, then an i64 in
    [0, 1000)). Median CUDA-event kernel_ms of 5 runs after 1 warm-up (sort plus the gathers of every column), and algorithmic bytes
    over time: the columns read once and written once in the new order.
  * pipelines, host clock around the whole action after a warm-up run over a tiny input:
      agg_collect   the aggbykey shape as a CSV file (--groups distinct 'k%07d' keys, two rows per key, i64 values) ->
                    aggregateByKey(sum) -> collect
      agg_tocsv     the same -> map -> tocsv
      u311_tocsv    tests/golden/311-service-requests-sf=1.csv replicated --n311 times -> mapColumn(fix_zip_codes) -> unique -> tocsv
    With --against DIR every pipeline runs in a fresh process per tree, alternating this tree with the tree at DIR (e.g. a build of
    the parent commit), --runs times, and the outputs (CSV bytes, collected rows) are compared by md5.
Prints one JSON object with the card's name and power limit; with --out it is also written to that file.

    python tools/hash_handoff_probe.py [--rows 10000000] [--groups 10000000] [--n311 50] [--runs 2] [--against DIR] [--out f.json]
"""
import argparse
import gzip
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


# ---- inputs -------------------------------------------------------------------------------------------------------------------
def agg_file(dirname: str, groups: int) -> str:
    """CSV (key, v): every one of `groups` keys 'k%07d' twice, in a seeded random order."""
    import numpy as np
    path = os.path.join(dirname, f"agg_{groups}.csv")
    if not os.path.exists(path):
        rng = np.random.default_rng(42)
        ids = rng.permutation(np.concatenate([np.arange(groups), np.arange(groups)]))
        vals = rng.integers(-1000, 1000, len(ids))
        digits = np.zeros((len(ids), 8), np.uint8)
        digits[:, 0] = ord("k")
        x = ids.copy()
        for p in range(7, 0, -1):
            digits[:, p] = ord("0") + x % 10
            x //= 10
        with open(path + ".tmp", "wb") as f:
            f.write(b"key,v\n")
            step = 1 << 20
            for lo in range(0, len(ids), step):
                keys = digits[lo:lo + step].tobytes()
                f.write(b"".join(keys[8 * i:8 * i + 8] + b"," + str(v).encode() + b"\n" for i, v in enumerate(vals[lo:lo + step].tolist())))
        os.replace(path + ".tmp", path)
    return path


def u311_file(dirname: str, n: int) -> str:
    path = os.path.join(dirname, f"311_{n}.csv")
    if not os.path.exists(path):
        data = gzip.open(os.path.join(ROOT, "tests", "golden", "311-service-requests-sf=1.csv.gz"), "rb").read()
        head, body = data.split(b"\n", 1)
        with open(path + ".tmp", "wb") as f:
            f.write(head + b"\n")
            for _ in range(n):
                f.write(body if body.endswith(b"\n") else body + b"\n")
        os.replace(path + ".tmp", path)
    return path


# ---- one pipeline in this process (the tree comes first on sys.path) ----------------------------------------------------------
def fix_zip_codes(zips):
    if not zips:
        return None
    s = zips[:5]
    return None if s == "00000" else s


def pipeline(name: str, path: str, out: str):
    import typing
    import tuplex_b200
    ctx = tuplex_b200.Context()
    t0 = time.perf_counter()
    if name == "u311_tocsv":
        ctx.csv(path, null_values=["Unspecified", "NO CLUE", "NA", "N/A", "0", ""], type_hints={0: typing.Optional[str]}) \
            .mapColumn("Incident Zip", fix_zip_codes).unique().tocsv(out)
        digest = hashlib.md5(open(out, "rb").read()).hexdigest()
    else:
        ds = ctx.csv(path).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["key"])
        if name == "agg_collect":
            rows = ds.collect()
            dt = time.perf_counter() - t0
            return dt, hashlib.md5(repr(rows).encode()).hexdigest(), getattr(ctx.metrics, "device_handoff_rows", None), len(rows)
        ds.map(lambda x: (x[0], x[1] * 2)).tocsv(out)
        digest = hashlib.md5(open(out, "rb").read()).hexdigest()
    dt = time.perf_counter() - t0
    return dt, digest, getattr(ctx.metrics, "device_handoff_rows", None), None


def worker(a):
    """--worker: warm up on a tiny input, then time one pipeline; prints one JSON line."""
    sys.path.insert(0, a.tree)
    with tempfile.TemporaryDirectory() as tmp:
        small = agg_file(tmp, 1000) if a.worker != "u311_tocsv" else u311_file(tmp, 1)
        pipeline(a.worker, small, os.path.join(tmp, "warm.csv"))
        dt, digest, handoff, n = pipeline(a.worker, a.input, os.path.join(tmp, "out.csv"))
    print(json.dumps({"s": round(dt, 3), "md5": digest, "handoff_rows": handoff, "rows": n}))


# ---- the sort alone -------------------------------------------------------------------------------------------------------------
def sort_alone(rows: int):
    sys.path.insert(0, ROOT)
    import numpy as np
    from tuplex_b200 import backend, frontend
    from tuplex_b200.backend import Column
    from tuplex_b200.ir import T_I64, T_STR
    rng = np.random.default_rng(7)
    backend.init([0])
    ids = rng.integers(0, rows, rows)
    lens = 8 + rng.integers(0, 9, rows)
    offs = np.zeros(rows + 1, np.uint32)
    np.cumsum(lens, out=offs[1:])
    data = rng.integers(ord("a"), ord("z") + 1, int(offs[-1])).astype(np.uint8)
    starts = offs[:-1].astype(np.int64)
    data[starts] = ord("k")
    x = ids.copy()
    for p in range(7, 0, -1):
        data[starts + p] = ord("0") + x % 10
        x //= 10
    s = Column(T_STR, data, offs)
    i64 = Column(T_I64, rng.integers(-(1 << 63), (1 << 63) - 1, rows, dtype=np.int64))
    small = Column(T_I64, rng.integers(0, 1000, rows).astype(np.int64))
    out = {}
    for name, cols in (("i64", [i64]), ("str_8_16", [s]), ("str_i64", [s, small])):
        sc = frontend.StageCompiler([c.type for c in cols], ["c%d" % k for k in range(len(cols))])
        st = backend.Stage(sc.finish_memory())
        res = st.run_host(0, cols, rows)
        nbytes = sum(int(res.info.out_str_bytes[c]) + (rows + 1) * 4 if c_.type == T_STR else rows * 8 for c, c_ in enumerate(cols)) * 2
        ms, launches = [], 0
        for k in range(6):
            o = res.sort_by_keys(len(cols))
            if k:
                ms.append(float(o.info.kernel_ms))
            launches = int(o.info.kernel_launches)
            o.free()
        med = statistics.median(ms)
        out[name] = {"kernel_ms": round(med, 3), "bytes": nbytes, "GB_per_s": round(nbytes / med / 1e6, 1), "launches": launches}
        res.free()
        st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--groups", type=int, default=10_000_000)
    ap.add_argument("--n311", type=int, default=50)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--against", default=None, help="another tree (e.g. the parent commit, built) to alternate the pipelines with")
    ap.add_argument("--only", choices=["sort", "pipelines"], default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--tree", default=ROOT, help=argparse.SUPPRESS)
    ap.add_argument("--input", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)
    res = {"card": card()}
    if a.only in (None, "sort"):
        res["sort_rows"] = a.rows
        res["sort"] = sort_alone(a.rows)
    if a.only in (None, "pipelines"):
        trees = [("this", ROOT)] + ([("against", os.path.abspath(a.against))] if a.against else [])
        with tempfile.TemporaryDirectory() as tmp:
            inputs = {"agg_collect": agg_file(tmp, a.groups), "u311_tocsv": u311_file(tmp, a.n311)}
            inputs["agg_tocsv"] = inputs["agg_collect"]
            for name, path in inputs.items():
                runs = {t: [] for t, _ in trees}
                for _ in range(a.runs):
                    for t, tree in trees:
                        q = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", name, "--tree", tree, "--input", path],
                                           capture_output=True, text=True, cwd=tree)
                        if q.returncode:
                            raise SystemExit(f"{name} on {tree} failed:\n{q.stderr[-3000:]}")
                        runs[t].append(json.loads(q.stdout.strip().splitlines()[-1]))
                res[name] = {t: {"s": [r["s"] for r in rs], "md5": sorted({r["md5"] for r in rs}), "handoff_rows": rs[-1]["handoff_rows"],
                                 "rows": rs[-1]["rows"]} for t, rs in runs.items()}
                if a.against:
                    res[name]["same_output"] = res[name]["this"]["md5"] == res[name]["against"]["md5"]
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
