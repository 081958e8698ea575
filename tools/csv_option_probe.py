"""Cost of an Option[str] column in the device CSV source (K6), on a 311-shaped input: the sf=1 Incident Zip fixture replicated
to about 1 GB, and a seeded variant of the same size with 10 % of its cells
emptied (written as a quoted empty cell, which matches the null value ""). Prints the card and its power limit, the median
parse_ms over several runs after warm-up with the zip column read as str and as Option[str], and the host clock of the whole
csv -> mapColumn(fix_zip_codes) -> unique pipeline (its device work ends in a synchronise inside collect).
usage: python tools/csv_option_probe.py [MB] [runs]"""
import gzip
import os
import random
import statistics
import subprocess
import sys
import tempfile
import time
import typing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import tuplex_b200  # noqa: E402
from tuplex_b200 import backend, ir  # noqa: E402

NULLS = ["Unspecified", "NO CLUE", "NA", "N/A", "0", ""]
OPT = ir.C["TPLX_T_OPTION"]


def fix_zip_codes(zips):
    if not zips:
        return None
    s = zips[:5]
    if s == "00000":
        return None
    else:
        return s


def inputs(mb: int):
    raw = gzip.open(os.path.join(ROOT, "tests", "golden", "311-service-requests-sf=1.csv.gz"), "rb").read()
    header, body = raw.split(b"\n", 1)
    reps = max(1, (mb << 20) // len(body))
    rng = random.Random(311)
    lines = body.split(b"\n")
    if lines[-1] == b"":
        lines.pop()
    # an emptied cell is written quoted: a bare empty line would be a blank line, which the row finder skips
    empty = b"\n".join(b'""' if rng.random() < 0.10 else ln for ln in lines) + b"\n"
    print(f"fixture body replicated {reps} times")
    return {"fixture": header + b"\n" + body * reps, "10pct_empty": header + b"\n" + empty * reps}


def main():
    mb = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    runs = int(sys.argv[2]) if len(sys.argv) > 2 else 7
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print("card:", card.strip().splitlines()[0] if card.strip() else "unknown")
    backend.init([0])
    for name, data in inputs(mb).items():
        arr = np.frombuffer(data, dtype=np.uint8)
        buf = backend.CsvBuffer(0, arr)
        for label, t in (("str", ir.T_STR), ("Option[str]", ir.T_STR | OPT)):
            times = []
            for it in range(2 + runs):  # two warm-up parses
                p = buf.parse([t], header=True, null_values=NULLS)
                info = p.info
                if it >= 2:
                    times.append(float(info.parse_ms))
                rows, bad, launches = int(info.n_rows), int(info.n_bad), int(info.kernel_launches)
                p.free()
            print(f"{name}: {len(data) / 1e9:.3f} GB, {rows} rows, zip as {label}: parse_ms median {statistics.median(times):.3f} "
                  f"(min {min(times):.3f}, max {max(times):.3f}, {runs} runs), bad rows {bad}, launches {launches}")
        buf.free()
        with tempfile.NamedTemporaryFile(suffix=".csv") as f:
            f.write(data)
            f.flush()
            for it in range(2):
                ctx = tuplex_b200.Context()
                t0 = time.perf_counter()
                out = ctx.csv(f.name, null_values=NULLS, type_hints={0: typing.Optional[str]}).mapColumn("Incident Zip", fix_zip_codes) \
                    .unique().collect()
                dt = time.perf_counter() - t0
                print(f"{name}: pipeline csv -> mapColumn -> unique (Option[str]) run {it}: {dt * 1e3:.1f} ms host clock, "
                      f"{len(out)} distinct, csv_bad_rows {ctx.metrics.csv_bad_rows}, exceptions {ctx.metrics.exceptions}, "
                      f"csv_parse_ms {ctx.metrics.csv_parse_ms:.3f}")


if __name__ == "__main__":
    main()
