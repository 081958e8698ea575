"""What pipelines through a join cost end to end, and what the block concatenation of a join's build side costs.

Pipelines, host clock around the whole run (sources read, stages, joins and the CSV sink; tocsv returns after the device has
finished):
  * logs: the reference's Apache logs pipeline on tests/golden/logs.sample.txt replicated to about --mb MB (as tools/text_probe.py
    builds it): text -> map(ParseWithStrip) -> join(bad IPs, tests/golden/bad_ips_all.txt) -> selectColumns -> tocsv;
  * flights: the flights-like pipeline of tests/test_flights_like.py (three joins, post-join stages) over --flights synthetic rows
    generated from a seed, -> tocsv. The tables are built before the clock starts.
Each pipeline first runs once over a tenth of its input to warm up (module loads, stage specialiser compiles), then --runs times.
  * concat: tplx_gpu_block_concat of the logs stage's per-chunk results (the parsed logs as one build-side block): device time
    (host clock around the call, which ends in a device synchronise), bytes of the concatenated columns, median of 5 after 1 warm-up.
Prints one JSON object (with the card's name and power limit and the md5 of each pipeline's CSV output); with --out it is also
written to that file.

    python tools/join_handoff_probe.py [--mb 1000] [--flights 2000000] [--runs 3] [--only logs|flights] [--data DIR] [--out f.json]
"""
import argparse
import gzip
import json
import os
import pickle
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
from logs_udfs import ParseWithStrip  # noqa: E402


def logs_file(dirname: str, mb: int) -> str:
    path = os.path.join(dirname, f"logs_{mb}.txt")
    if not os.path.exists(path):
        sample = gzip.open(os.path.join(ROOT, "tests", "golden", "logs.sample.txt.gz"), "rb").read()
        with open(path + ".tmp", "wb") as f:
            for _ in range(max(1, mb * 1000 * 1000 // len(sample))):
                f.write(sample)
        os.replace(path + ".tmp", path)
    return path


def ips_file(dirname: str) -> str:
    path = os.path.join(dirname, "bad_ips_all.txt")
    if not os.path.exists(path):
        open(path, "wb").write(gzip.open(os.path.join(ROOT, "tests", "golden", "bad_ips_all.txt.gz"), "rb").read())
    return path


def flights_tables(dirname: str, n: int):
    path = os.path.join(dirname, f"flights_{n}.pkl")
    if not os.path.exists(path):
        import test_flights_like as fl
        with open(path + ".tmp", "wb") as f:
            pickle.dump(fl._tables(n, 11), f)
        os.replace(path + ".tmp", path)
    with open(path, "rb") as f:
        return pickle.load(f)


def run_logs(logs: str, ips: str, out: str):
    ctx = tuplex_b200.Context()
    ds = ctx.text(logs).map(ParseWithStrip).join(ctx.csv(ips), "ip", "BadIPs").selectColumns(["ip", "endpoint"])
    t0 = time.perf_counter()
    ds.tocsv(out)
    return time.perf_counter() - t0, ctx


def run_flights(tables, out: str):
    import test_flights_like as fl
    flights, carriers, airports = tables
    c = tuplex_b200.Context()
    t0 = time.perf_counter()
    df = c.parallelize(flights, columns=fl.F_COLS)
    df = df.withColumn('OriginCity', lambda x: x['OriginCityName'][:x['OriginCityName'].rfind(',')].strip())
    df = df.withColumn('OriginState', lambda x: x['OriginCityName'][x['OriginCityName'].rfind(',') + 1:].strip())
    df = df.withColumn('DestCity', lambda x: x['DestCityName'][:x['DestCityName'].rfind(',')].strip())
    df = df.mapColumn('CrsArrTime', lambda x: '{:02}:{:02}'.format(int(x / 100), x % 100) if x else None)
    df = df.withColumn('CancellationCode', fl.cleanCode)
    df = df.mapColumn('Diverted', lambda x: True if x > 0 else False)
    df = df.withColumn('CancellationReason', fl.divertedUDF)
    df = df.withColumn('ActualElapsedTime', fl.fillInTimesUDF).ignore(TypeError)
    dc = c.parallelize(carriers, columns=fl.C_COLS)
    dc = dc.withColumn('AirlineName', lambda x: x['Description'][:x['Description'].rfind('(')].strip())
    dc = dc.withColumn('AirlineYearFounded', lambda x: int(x['Description'][x['Description'].rfind('(') + 1:x['Description'].rfind('-')]))
    dc = dc.withColumn('AirlineYearDefunct', fl.extractDefunctYear)
    da = c.parallelize(airports, columns=fl.A_COLS)
    dall = df.join(dc, 'OpUniqueCarrier', 'Code')
    dall = dall.leftJoin(da, 'Origin', 'IATACode', prefixes=(None, 'Origin'))
    dall = dall.leftJoin(da, 'Dest', 'IATACode', prefixes=(None, 'Dest'))
    dall = dall.mapColumn('Distance', lambda x: x / 0.00062137119224)
    dall = dall.mapColumn('AirlineName', lambda s: s.replace('Inc.', '').replace('LLC', '').replace('Co.', '').strip())
    dall = dall.renameColumn('AirlineName', 'CarrierName').renameColumn('Origin', 'OriginAirportIATACode')
    dall = dall.filter(fl.filterDefunctFlights)
    dall.tocsv(out)
    return time.perf_counter() - t0, c


def concat(logs: str):
    """Block.concat of the parsed logs' per-chunk results (only where the tree has it)."""
    if not hasattr(backend.Block, "concat"):
        return None
    ctx = tuplex_b200.Context()
    ds = ctx.text(logs)
    ds._source.chunk_bytes = 128 << 20  # several parse chunks, so several stage results to concatenate
    rows, _ = ds.map(ParseWithStrip)._execute(handoff=True)
    parts = [p.as_block(len(rows.types)) for p in rows.parts]
    times = []
    for k in range(6):
        t0 = time.perf_counter()
        b = backend.Block.concat(parts)
        dt = time.perf_counter() - t0
        b.free()
        if k:
            times.append(dt * 1e3)
    nbytes = sum(int(p.info.out_str_bytes[c]) + int(p.info.n_out_rows) * 4 if t == backend.T_STR else int(p.info.n_out_rows) * 8
                 for p in rows.parts for c, t in enumerate(rows.types))
    ms = statistics.median(times)
    return {"parts": len(parts), "rows": rows.n_rows, "bytes": nbytes, "ms": ms, "GB_per_s": nbytes / ms / 1e6}


def md5(path: str) -> str:
    import hashlib
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=1000)
    ap.add_argument("--flights", type=int, default=2000000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--only", choices=["logs", "flights"], default=None)
    ap.add_argument("--data", default=None, help="directory for the generated inputs (kept between invocations)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    data = a.data or tempfile.mkdtemp()
    os.makedirs(data, exist_ok=True)
    res = {"tree": ROOT, "card": card()}
    with tempfile.TemporaryDirectory() as tmp:
        if a.only in (None, "logs"):
            logs, ips = logs_file(data, a.mb), ips_file(data)
            res["logs_mb"] = os.path.getsize(logs) / 1e6
            run_logs(logs_file(data, max(1, a.mb // 10)), ips, os.path.join(tmp, "warm.csv"))
            ts = [run_logs(logs, ips, os.path.join(tmp, f"logs{k}.csv")) for k in range(a.runs)]
            res["logs_s"] = [round(t, 3) for t, _ in ts]
            res["logs_handoff_rows"] = getattr(ts[-1][1].metrics, "device_handoff_rows", None)
            res["logs_md5"] = md5(os.path.join(tmp, f"logs{a.runs - 1}.csv"))
            res["concat"] = concat(logs)
        if a.only in (None, "flights"):
            tables = flights_tables(data, a.flights)
            res["flights_rows"] = a.flights
            run_flights(flights_tables(data, max(1, a.flights // 10)), os.path.join(tmp, "warm.csv"))
            ts = [run_flights(tables, os.path.join(tmp, f"fl{k}.csv")) for k in range(a.runs)]
            res["flights_s"] = [round(t, 3) for t, _ in ts]
            res["flights_handoff_rows"] = getattr(ts[-1][1].metrics, "device_handoff_rows", None)
            res["flights_md5"] = md5(os.path.join(tmp, f"fl{a.runs - 1}.csv"))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
