"""Join inputs and outputs that stay on the device: tplx_gpu_block_concat against numpy concatenation of its parts, and pipelines
through a join against a nested-loop join of the CPython rows. Every pipeline test also asserts which path ran, through
ctx.metrics.device_handoff_rows: the rows each join took from a stage result or an upstream join, plus the join output rows the next
stage, join or tocsv took on the device; zero where the host path must run."""
import gzip
import os
import random

import numpy as np
import pytest

import tuplex_b200
from tuplex_b200 import backend, dataset, frontend
from tuplex_b200.backend import Column
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR
from tuplex_b200.textsource import read_lines

from logs_udfs import ParseWithStrip

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


# ---- tplx_gpu_block_concat ------------------------------------------------------------------------------------------------
def _column(rng, t, n):
    if t == T_STR:
        lens = rng.integers(0, 12, n)
        offs = np.zeros(n + 1, np.uint32)
        np.cumsum(lens, out=offs[1:])
        # NULs, invalid UTF-8 (0xFF, lone continuation bytes) and ASCII; lengths 0..11 put string starts at every offset mod 16
        alphabet = np.frombuffer(b"\x00\xff\x80abcXYZ,\"\n", np.uint8)
        return Column(T_STR, alphabet[rng.integers(0, len(alphabet), int(offs[-1]))], offs)
    if t == T_F64:
        return Column(T_F64, rng.standard_normal(n) * 1e6)
    if t == T_BOOL:
        return Column(T_BOOL, rng.integers(0, 2, n).astype(np.int64))
    return Column(T_I64, rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64))


def _fetch(block: backend.Block, t: int, option: bool):
    """(values or (bytes, offsets)) of a one-column block, read back through an identity stage."""
    sc = frontend.StageCompiler([t], ["c"], [0] if option else [])
    sc.add_map(lambda x: x, 100001)
    st = backend.Stage(sc.finish_memory())
    res = st.run(block)
    assert int(res.info.n_out_rows) == block.n_rows and int(res.info.n_exceptions) == 0
    col = res.column(0)
    out = (col.data.tobytes(), col.offsets.tolist()) if t == T_STR else col.data.copy()
    res.free()
    st.close()
    return out


SIZES = [0, 1, 31, 32, 33, (1 << 21) + 5]


@pytest.mark.parametrize("option", [False, True], ids=["plain", "option"])
@pytest.mark.parametrize("t", [T_I64, T_F64, T_BOOL, T_STR], ids=["i64", "f64", "bool", "str"])
def test_concat_matches_numpy(gpu, t, option):
    rng = np.random.default_rng(7 + t)
    sizes = SIZES + [33, 0, 1, 32]
    random.Random(t).shuffle(sizes)
    cols, present = [], []
    for k, n in enumerate(sizes):
        col = _column(rng, t, n)
        pres = np.ones(n, bool)
        if option and k % 3 != 1:  # bitmaps on some parts only
            pres = rng.random(n) < 0.7
            words = backend.pack_valid(pres)
            if n & 31:  # garbage past the part's row count: must not reach the output
                words[-1] |= np.uint32(0xFFFFFFFF) << np.uint32(n & 31)
            col.valid = words
        cols.append(col)
        present.append(pres)
    parts = [backend.Block.upload(0, [c], len(c)) for c in cols]
    out = backend.Block.concat(parts)
    for p in parts:
        p.free()  # the output owns its memory
    n = sum(sizes)
    assert out.n_rows == n
    got = _fetch(out, t, option)
    if t == T_STR:
        want_bytes = b"".join(c.data.tobytes() for c in cols)
        base = np.cumsum([0] + [int(c.offsets[-1]) for c in cols])
        want_offs = np.concatenate([c.offsets[:-1].astype(np.int64) + b for c, b in zip(cols, base)] + [np.array([base[-1]])])
        assert got[0] == want_bytes and got[1] == want_offs.tolist()
    else:
        want = np.concatenate([c.data for c in cols])
        assert got.tobytes() == want.tobytes()
    words = out.validity(0)
    if option:
        assert words is not None and words.tolist() == backend.pack_valid(np.concatenate(present)).tolist()  # tail bits zero
    else:
        assert words is None
    out.free()


def test_concat_several_columns_zero_parts_and_errors(gpu):
    rng = np.random.default_rng(3)
    a = [_column(rng, T_STR, 40), _column(rng, T_I64, 40)]
    b = [_column(rng, T_STR, 7), _column(rng, T_I64, 7)]
    pa, pb = backend.Block.upload(0, a, 40), backend.Block.upload(0, b, 7)
    out = backend.Block.concat([pa, pb])
    assert out.n_rows == 47 and out.validity(0) is None and out.validity(1) is None
    empty = backend.Block.concat([])
    assert empty.n_rows == 0
    with pytest.raises(backend.GpuBackendError, match="types"):
        backend.Block.concat([pa, backend.Block.upload(0, [b[1], b[0]], 7)])
    with pytest.raises(backend.GpuBackendError, match="column counts"):
        backend.Block.concat([pa, backend.Block.upload(0, b[:1], 7)])
    # a string column over 4 GiB is refused before anything is read (the byte counts are the parts' own)
    big = [backend.Block.wrap_device(0, [(T_STR, 16, 16, 3 << 30)], 0) for _ in range(2)]
    with pytest.raises(backend.GpuBackendError, match="4 GiB"):
        backend.Block.concat(big)
    for x in (pa, pb, out, empty):
        x.free()


# ---- pipelines ------------------------------------------------------------------------------------------------------------
def _ctx(**kw):
    conf = {"tuplex.gpu.blockRows": 64}
    conf.update(kw)
    return tuplex_b200.Context(conf)


def _nested_join(L, li, R, ri, left_outer=False):
    out = []
    for l in L:
        ms = [r for r in R if r[ri] == l[li] and type(r[ri]) is type(l[li])]
        out += [tuple(v for i, v in enumerate(l) if i != li) + (l[li],) + tuple(v for i, v in enumerate(r) if i != ri) for r in ms]
        if not ms and left_outer:
            out.append(tuple(v for i, v in enumerate(l) if i != li) + (l[li],) + (None,) * (len(R[0]) - 1))
    return out


def _golden(tmp_path, name):
    p = tmp_path / name
    p.write_bytes(gzip.open(os.path.join(HERE, "golden", name + ".gz"), "rb").read())
    return str(p)


def _parsed_logs(path):
    out = []
    for ln in read_lines([path], print):
        try:
            out.append(ParseWithStrip(ln))
        except Exception:  # noqa: BLE001 — the row raised: dropped like an unresolved exception row
            pass
    return out


def test_apache_dev(gpu, tmp_path):
    logs, ips = _golden(tmp_path, "logs.sample.txt"), _golden(tmp_path, "bad_ips_all.txt")
    ctx = tuplex_b200.Context()
    rows = ctx.text(logs).map(ParseWithStrip).join(ctx.csv(ips), "ip", "BadIPs").collect()
    parsed = _parsed_logs(logs)
    bad = read_lines([ips], print)[1:]
    names = list(parsed[0].keys())
    want = _nested_join([tuple(d.values()) for d in parsed], names.index("ip"), [(b,) for b in bad], 0)
    assert len(rows) == 3437 and rows == want
    assert ctx.metrics.device_handoff_rows == len(parsed) + len(bad)


def test_null_value_apache_tocsv(gpu, tmp_path):
    logs, ips = _golden(tmp_path, "logs.sample.txt"), _golden(tmp_path, "ip_blacklist.csv")
    ctx = tuplex_b200.Context()
    out = str(tmp_path / "logs.csv")
    ds = ctx.text(logs).map(ParseWithStrip).join(ctx.csv(ips), "ip", "BadIPs")
    ds.selectColumns(["ip", "endpoint"]).tocsv(out)
    assert open(out, "rb").read() == b"ip,endpoint\n1.1.209.108,/research/finance/\n"
    n_ips = len(read_lines([ips], print)) - 1  # header
    assert ctx.metrics.device_handoff_rows == len(_parsed_logs(logs)) + n_ips + 1  # both sides, then the join's one row


def test_flights_like_several_blocks_per_side(gpu):
    import test_flights_like as fl
    flights, carriers, airports = fl._tables(3000, 5)
    want, want_names = fl._expected(flights, carriers, airports)
    c = tuplex_b200.Context({"tuplex.gpu.blockRows": 2})
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
    assert dall.columns == want_names
    assert dall.collect() == want
    # handed-off rows: flights and carriers after their stages, each join's output into the next join / the post-join stage, and
    # the airport table (an identity stage) twice
    rows, names = list(flights), list(fl.F_COLS)
    for kind, name, fn in [("withColumn", "OriginCity", lambda x: x['OriginCityName'][:x['OriginCityName'].rfind(',')].strip()),
                           ("withColumn", "OriginState", lambda x: x['OriginCityName'][x['OriginCityName'].rfind(',') + 1:].strip()),
                           ("withColumn", "DestCity", lambda x: x['DestCityName'][:x['DestCityName'].rfind(',')].strip()),
                           ("mapColumn", "CrsArrTime", lambda x: '{:02}:{:02}'.format(int(x / 100), x % 100) if x else None),
                           ("withColumn", "CancellationCode", fl.cleanCode), ("mapColumn", "Diverted", lambda x: True if x > 0 else False),
                           ("withColumn", "CancellationReason", fl.divertedUDF), ("withColumn", "ActualElapsedTime", fl.fillInTimesUDF)]:
        rows, names = fl._apply(rows, names, kind, name, fn)
    crow, cn = list(carriers), list(fl.C_COLS)
    for kind, name, fn in [("withColumn", "AirlineName", lambda x: x['Description'][:x['Description'].rfind('(')].strip()),
                           ("withColumn", "AirlineYearFounded", lambda x: int(x['Description'][x['Description'].rfind('(') + 1:x['Description'].rfind('-')])),
                           ("withColumn", "AirlineYearDefunct", fl.extractDefunctYear)]:
        crow, cn = fl._apply(crow, cn, kind, name, fn)
    j1 = [r for r in rows for k in crow if k[0] == r[1]]
    j2 = j1  # left joins keep every row: the airport table has one row per code
    assert c.metrics.device_handoff_rows == len(rows) + len(crow) + len(j1) + len(airports) + len(j2) + len(airports) + len(j2)
    assert getattr(c.metrics, "join_concat_ms", 0) > 0  # the build sides spanned several blocks


def _lr(ctx):
    L = [(i, f"v{i}", i % 7 == 0 or None) for i in range(200)]
    R = [(i, f"r{i}" if i % 5 else None) for i in range(0, 300, 3)]
    dl = ctx.parallelize(L, columns=["k", "a", "f"]).withColumn("b", lambda x: x["k"] * 2)
    dr = ctx.parallelize(R, columns=["k", "s"]).withColumn("t", lambda x: x["k"] + 1)
    Lx = [r + (r[0] * 2,) for r in L]
    Rx = [r + (r[0] + 1,) for r in R]
    return dl, dr, Lx, Rx


def test_left_join_none_columns_feed_a_stage(gpu):
    ctx = _ctx()
    dl, dr, L, R = _lr(ctx)
    ds = dl.leftJoin(dr, "k", "k").map(lambda x: (x["k"], x["s"] if x["s"] is not None else "none", x["t"] is None))
    got = ds.collect()
    j = _nested_join(L, 0, R, 0, left_outer=True)  # a, f, b, k, s, t
    assert got == [(r[3], r[4] if r[4] is not None else "none", r[5] is None) for r in j]
    assert ctx.metrics.device_handoff_rows == len(L) + len(R) + len(j)


def test_pre_join_resolved_rows(gpu):
    """Rows resolved into the stage's schema are merged on the device (K9); resolved rows of another type send that side home."""
    for fits in (True, False):
        ctx = _ctx()
        dl = ctx.parallelize([(i, i % 5) for i in range(150)], columns=["k", "d"]).withColumn("q", lambda x: 100 // x["d"])
        dl = dl.resolve(ZeroDivisionError, (lambda x: -1) if fits else (lambda x: "bad"))
        dr = ctx.parallelize([(i, str(i)) for i in range(0, 150, 2)], columns=["k", "s"]).withColumn("u", lambda x: x["s"] + "!")
        got = dl.join(dr, "k", "k").collect()
        L = [(i, i % 5, (100 // (i % 5)) if i % 5 else (-1 if fits else "bad")) for i in range(150)]
        R = [(i, str(i), str(i) + "!") for i in range(0, 150, 2)]
        assert got == _nested_join(L, 0, R, 0)
        assert ctx.metrics.device_handoff_rows == ((len(L) + len(R)) if fits else 0)  # a host side with fallback rows: host path


@pytest.mark.parametrize("mode", ["raise", "resolve", "ignore"])
def test_post_join_stage_raises(gpu, mode):
    ctx = _ctx()
    dl, dr, L, R = _lr(ctx)
    ds = dl.join(dr, "k", "k").map(lambda x: 1000 // (x["k"] % 4))
    if mode == "resolve":
        ds = ds.resolve(ZeroDivisionError, lambda x: -7)
    elif mode == "ignore":
        ds = ds.ignore(ZeroDivisionError)
    got = ds.collect()
    j = _nested_join(L, 0, R, 0)
    want = [1000 // (r[3] % 4) if r[3] % 4 else -7 for r in j if r[3] % 4 or mode == "resolve"]
    assert got == want
    if mode == "raise":
        assert sum(ds.exception_counts.values()) == sum(1 for r in j if r[3] % 4 == 0)
    assert ctx.metrics.device_handoff_rows == len(L) + len(R) + len(j)


def test_join_then_endpoints(gpu):
    for end in ("aggregate", "aggregateByKey", "unique"):
        ctx = _ctx()
        dl, dr, L, R = _lr(ctx)
        j = _nested_join(L, 0, R, 0)
        ds = dl.join(dr, "k", "k")
        if end == "aggregate":
            got = ds.aggregate(lambda a, b: a + b, lambda a, x: a + x["t"], 0).collect()
            want = [sum(r[5] for r in j)]
        elif end == "aggregateByKey":
            got = ds.map(lambda x: (x["k"] % 3, x["t"])).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x[1], 0, [0]).collect()
            want = sorted({(r[3] % 3, sum(q[5] for q in j if q[3] % 3 == r[3] % 3)) for r in j})
            got = sorted(got)
        else:
            got = sorted(ds.map(lambda x: x["k"] % 6).unique().collect())
            want = sorted({r[3] % 6 for r in j})
        assert got == want, end
        assert ctx.metrics.device_handoff_rows == len(L) + len(R) + len(j), end


def test_join_tocsv_equals_host_writer(gpu, tmp_path):
    ctx = _ctx()
    dl, dr, L, R = _lr(ctx)
    out = str(tmp_path / "j.csv")
    dl.leftJoin(dr, "k", "k").tocsv(out, null_value="NA")
    j = _nested_join(L, 0, R, 0, left_outer=True)
    names = ["a", "f", "b", "k", "s", "t"]
    want = ",".join(names) + "\n" + "".join(",".join(dataset._csv_cell(v, "NA") for v in r) + "\n" for r in j)
    assert open(out, "rb").read() == want.encode()
    assert ctx.metrics.device_handoff_rows == len(L) + len(R) + len(j)


def test_empty_side_and_no_match(gpu):
    ctx = _ctx()
    dl, dr, L, R = _lr(ctx)
    assert dl.filter(lambda x: x["k"] < 0).join(dr, "k", "k").collect() == []
    assert ctx.metrics.device_handoff_rows == len(R)
    ctx = _ctx()
    dl, dr, L, R = _lr(ctx)
    got = dl.leftJoin(dr.filter(lambda x: x["k"] < 0), "k", "k").map(lambda x: (x["k"], x["a"])).collect()
    assert got == [(r[0], r[1]) for r in L]
    assert ctx.metrics.device_handoff_rows == len(L)  # the right columns are None in every row: the stage runs on host rows
    ctx = _ctx()
    dl, dr, L, R = _lr(ctx)
    got = dl.join(dr.mapColumn("k", lambda k: k + 100000), "k", "k").collect()
    assert got == []
    assert ctx.metrics.device_handoff_rows == len(L) + len(R)


class _NoCompiler:
    def __init__(self, *args, **kwargs):
        raise frontend.UnsupportedUDF("every stage on the CPython path")


@pytest.mark.parametrize("cond", ["devices", "no_option", "fallback", "interpreter", "f64_key"])
def test_host_path_conditions(gpu, cond, monkeypatch):
    conf = {"devices": {"tuplex.gpu.devices": "0,0"}, "no_option": {"tuplex.gpu.optionColumns": "false"}}.get(cond, {})
    ctx = _ctx(**conf)
    L = [(i, f"v{i}") for i in range(100)]
    R = [(i, i * 0.5) for i in range(0, 100, 4)]
    if cond == "fallback":  # rows outside the normal-case schema on both sides
        L, R = L + [("x", "y")], R + [("z", 1)]
    if cond == "interpreter":
        monkeypatch.setattr(dataset, "StageCompiler", _NoCompiler)
    if cond == "f64_key":
        L = [(float(k), v) for k, v in L]
        R = [(float(k), v) for k, v in R]
    dl = ctx.parallelize(L, columns=["k", "a"]).withColumn("c", lambda x: x["a"])
    dr = ctx.parallelize(R, columns=["k", "b"]).withColumn("d", lambda x: x["b"])
    got = dl.join(dr, "k", "k").map(lambda x: (x["k"], x["c"], x["d"])).collect()
    Lx = [r + (r[1],) for r in L]
    Rx = [r + (r[1],) for r in R]
    assert got == [(r[2], r[1], r[4]) for r in _nested_join(Lx, 0, Rx, 0)]
    assert ctx.metrics.device_handoff_rows == 0


def test_none_in_every_row_goes_home(gpu):
    """A join output column that is None in every row is typed from its values on the host path; the stage after the join then
    runs over host rows (the join's sides still came from the device)."""
    ctx = _ctx()
    dl = ctx.parallelize([(i, f"v{i}") for i in range(50)], columns=["k", "a"]).withColumn("b", lambda x: x["k"])
    dr = ctx.parallelize([(1000, "x")], columns=["k", "s"]).withColumn("t", lambda x: x["s"])
    got = dl.leftJoin(dr, "k", "k").map(lambda x: (x["k"], x["s"] is None)).collect()
    assert got == [(i, True) for i in range(50)]
    assert ctx.metrics.device_handoff_rows == 50 + 1
