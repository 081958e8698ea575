"""What a stage split at a CPython operator costs end to end, against the tree at --against (e.g. a build of the parent commit, where
such a stage runs wholly in CPython). Every pipeline runs in a fresh process per tree, the trees alternating, --runs times; the host
clock covers the whole action (planning, parse, stages, CPython calls, join, write) after a warm-up over a tiny input, and the
outputs are compared by md5.

  logs      the logs fixture replicated to --logs-mb MB: text -> map(ParseWithStrip) -> mapColumn("endpoint", re.sub with a fixed
            replacement: the reference's randomize_udf made deterministic) -> join(bad IPs) -> tocsv
  zillow    the Z1 fixture replicated --zillow-k times as CSV: Z1 with one more withColumn("price_k", round(price / 1000, 1)) -> tocsv
  flights   the flights-like tables of tests/test_flights_like.py (--flights rows): airports with mapColumn(string.capwords) on
            their city, joined to the flights -> tocsv
Prints one JSON object with the card's name and power limit; with --out it is also written to that file.

    python tools/split_probe.py [--logs-mb 1000] [--zillow-k 2000] [--flights 2000000] [--runs 2] [--against DIR] [--out f.json]
"""
import argparse
import gzip
import hashlib
import json
import os
import pickle
import re
import string
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
def _replicated(dirname: str, name: str, golden: str, times: int, header: bool) -> str:
    path = os.path.join(dirname, name)
    if not os.path.exists(path):
        data = gzip.open(os.path.join(ROOT, "tests", "golden", golden), "rb").read()
        head, body = data.split(b"\n", 1) if header else (b"", data)
        body = body if body.endswith(b"\n") else body + b"\n"
        with open(path + ".tmp", "wb") as f:
            if header:
                f.write(head + b"\n")
            for _ in range(max(1, times)):
                f.write(body)
        os.replace(path + ".tmp", path)
    return path


def inputs(dirname: str, a, small: bool = False) -> dict:
    sample = len(gzip.open(os.path.join(ROOT, "tests", "golden", "logs.sample.txt.gz"), "rb").read())
    logs_times = 1 if small else a.logs_mb * 1000 * 1000 // sample
    tag = "small" if small else "big"
    ips = _replicated(dirname, "bad_ips.txt", "bad_ips_all.txt.gz", 1, False)
    flights = os.path.join(dirname, f"flights_{tag}.pkl")
    if not os.path.exists(flights):
        sys.path += [p for p in (ROOT, os.path.join(ROOT, "tests")) if p not in sys.path]  # after a worker's tree
        import test_flights_like as fl
        with open(flights, "wb") as f:
            pickle.dump(fl._tables(1000 if small else a.flights, 11), f)
    return {"logs": (_replicated(dirname, f"logs_{tag}.txt", "logs.sample.txt.gz", logs_times, False), ips),
            "zillow": (_replicated(dirname, f"zillow_{tag}.csv", "zillow_noexc.csv.gz", 1 if small else a.zillow_k, True),),
            "flights": (flights,)}


# ---- one pipeline in this process (the tree comes first on sys.path) ----------------------------------------------------------
def fixed_randomize(x):
    return re.sub("^/~[^/]+", "/~" + "ABCDEFGHIJ", x)


def pipeline(name: str, paths, out: str):
    import tuplex_b200
    from tuplex_b200 import workloads
    ctx = tuplex_b200.Context()
    t0 = time.perf_counter()
    if name == "logs":
        from logs_udfs import ParseWithStrip
        logs, ips = paths
        (ctx.text(logs).map(ParseWithStrip).mapColumn("endpoint", fixed_randomize)
         .join(ctx.csv(ips), "ip", "BadIPs").tocsv(out))
    elif name == "zillow":
        ds = workloads.zillow_pipeline(ctx.csv(paths[0]))
        ds.withColumn("price_k", lambda x: round(x["price"] / 1000, 1)).tocsv(out)
    else:
        import test_flights_like as fl
        with open(paths[0], "rb") as f:
            flights, carriers, airports = pickle.load(f)
        da = ctx.parallelize(airports, columns=fl.A_COLS).withColumn("Lat", lambda x: x["LatitudeDecimal"] * 1.0) \
            .mapColumn("AirportCity", lambda s: string.capwords(s))
        df = ctx.parallelize(flights, columns=fl.F_COLS)
        df.leftJoin(da, "Origin", "IATACode", prefixes=(None, "Origin")).tocsv(out)
    dt = time.perf_counter() - t0
    return dt, hashlib.md5(open(out, "rb").read()).hexdigest(), getattr(ctx.metrics, "split_stages", None), \
        getattr(ctx.metrics, "interpreter_values", None)


def worker(a):
    """--worker: warm up on a tiny input, then time one pipeline; prints one JSON line."""
    sys.path.insert(0, a.tree)
    sys.path.insert(1, os.path.join(ROOT, "tests"))
    with tempfile.TemporaryDirectory() as tmp:
        pipeline(a.worker, inputs(tmp, a, small=True)[a.worker], os.path.join(tmp, "warm.csv"))
        dt, digest, splits, values = pipeline(a.worker, json.loads(a.input), os.path.join(tmp, "out.csv"))
    print(json.dumps({"s": round(dt, 3), "md5": digest, "split_stages": splits, "interpreter_values": values}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs-mb", type=int, default=1000)
    ap.add_argument("--zillow-k", type=int, default=2000)
    ap.add_argument("--flights", type=int, default=2_000_000)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--against", default=None, help="another tree (e.g. the parent commit, built) to alternate the pipelines with")
    ap.add_argument("--only", choices=["logs", "zillow", "flights"], default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--tree", default=ROOT, help=argparse.SUPPRESS)
    ap.add_argument("--input", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a)
    res = {"card": card()}
    trees = [("this", ROOT)] + ([("against", os.path.abspath(a.against))] if a.against else [])
    with tempfile.TemporaryDirectory() as tmp:
        for name, paths in inputs(tmp, a).items():
            if a.only not in (None, name):
                continue
            runs = {t: [] for t, _ in trees}
            for _ in range(a.runs):
                for t, tree in trees:
                    q = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", name, "--tree", tree, "--input", json.dumps(paths),
                                        "--logs-mb", str(a.logs_mb), "--zillow-k", str(a.zillow_k), "--flights", str(a.flights)],
                                       capture_output=True, text=True, cwd=tree)
                    if q.returncode:
                        raise SystemExit(f"{name} on {tree} failed:\n{q.stderr[-3000:]}")
                    runs[t].append(json.loads(q.stdout.strip().splitlines()[-1]))
                    print(name, t, runs[t][-1], file=sys.stderr, flush=True)  # progress: a run of the CPython path takes minutes
            res[name] = {t: {"s": [r["s"] for r in rs], "md5": sorted({r["md5"] for r in rs}), "split_stages": rs[-1]["split_stages"],
                             "interpreter_values": rs[-1]["interpreter_values"]} for t, rs in runs.items()}
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
