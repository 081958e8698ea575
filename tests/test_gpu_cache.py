"""DataSet.cache() on the device: tplx_gpu_block_stats and tplx_gpu_block_concat_pieces against numpy, then cached pipelines
against `ref`, the host dataset the same rows make (ctx._dataset_from_rows over ds._execute()). Every case asserts which path ran
through ctx.metrics.cache_rows (rows placed in device caches; 0 where the host path is required)."""
import gc
import gzip
import hashlib
import os
import random
import typing

import numpy as np
import pytest

import tuplex_b200
from tuplex_b200 import backend, dataset, frontend, workloads
from tuplex_b200.backend import Column
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR

from test_gpu_join_handoff import _column, _golden, _fetch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


# ---- tplx_gpu_block_stats and tplx_gpu_block_concat_pieces ---------------------------------------------------------------------
def _invalid(col: Column):
    raw, o = col.data.tobytes(), col.offsets
    return sum(raw[o[i]:o[i + 1]].decode("utf-8", "replace").encode() != raw[o[i]:o[i + 1]] for i in range(len(o) - 1))


def _with_bitmap(rng, col, n, density):
    pres = rng.random(n) < density
    words = backend.pack_valid(pres)
    if n & 31:  # garbage past the row count
        words[-1] |= np.uint32(0xFFFFFFFF) << np.uint32(n & 31)
    col.valid = words
    return pres


@pytest.mark.parametrize("t", [T_I64, T_F64, T_BOOL, T_STR], ids=["i64", "f64", "bool", "str"])
def test_stats_and_ranged_concat_match_numpy(gpu, t):
    rng = np.random.default_rng(11 + t)
    sizes = [0, 1, 31, 32, 33, 70, (1 << 21) + 5, 33, 1]
    cols, pres = [], []
    for k, n in enumerate(sizes):
        col = _column(rng, t, n)
        p = np.ones(n, bool) if k % 3 == 1 else _with_bitmap(rng, col, n, 0.6)
        if k % 3 == 1:
            col.valid = None
        cols.append(col)
        pres.append(p)
    blocks = [backend.Block.upload(0, [c], len(c)) for c in cols]
    for b, c, p in zip(blocks, cols, pres):
        none, bad = b.stats()
        assert none == [int((~p).sum())]
        assert bad == [_invalid(c) if t == T_STR else 0]
    # pieces starting at every row offset mod 32, cut across the parts; then one output block per flag
    pieces = []
    for k, (b, n) in enumerate(zip(blocks, sizes)):
        f = min(k % 32 + (k * 7) % 5, n)
        pieces.append((b, f, max(0, n - f - (k % 3))))
    pieces += [(blocks[6], r, 37) for r in range(0, 64 * 37, 37)]  # first rows at every offset mod 32 of one block
    idx = [next(i for i, x in enumerate(blocks) if x is b) for b, _, _ in pieces]
    want_pres = np.concatenate([pres[i][f:f + n] for i, (_, f, n) in zip(idx, pieces)])
    for flag in (0, backend.CONCAT_DROP_VALID, backend.CONCAT_ALL_NONE) + ((backend.CONCAT_UTF8,) if t == T_STR else ()):
        out = backend.Block.concat_pieces(pieces, [flag])
        assert out.n_rows == sum(n for _, _, n in pieces)
        got = out.column(0, T_I64 if flag == backend.CONCAT_ALL_NONE else t)
        if flag == backend.CONCAT_ALL_NONE:
            assert got.data.tolist() == [0] * out.n_rows and not got.present().any()
        else:
            if t == T_STR:
                strs = [cols[i].data[int(cols[i].offsets[r]):int(cols[i].offsets[r + 1])].tobytes() for i, (_, f, n) in zip(idx, pieces)
                        for r in range(f, f + n)]
                if flag == backend.CONCAT_UTF8:
                    strs = [s.decode("utf-8", "replace").encode() for s in strs]
                offs = np.zeros(len(strs) + 1, np.int64)
                np.cumsum([len(s) for s in strs], out=offs[1:])
                assert got.data.tobytes() == b"".join(strs) and got.offsets.tolist() == offs.tolist()
            else:
                want = np.concatenate([cols[i].data[f:f + n] for i, (_, f, n) in zip(idx, pieces)])
                assert got.data.tobytes() == want.tobytes()
            if flag == backend.CONCAT_DROP_VALID:
                assert got.valid is None
            else:
                assert got.valid.tolist() == backend.pack_valid(want_pres).tolist()
                assert out.validity(0).tolist() == got.valid.tolist()  # tail bits are zero
                none, _ = out.stats()
                assert none == [int((~want_pres).sum())]
        if flag == backend.CONCAT_UTF8:
            assert out.stats()[1] == [0]
            assert _fetch(out, t, True)[0] == got.data.tobytes()  # a stage reads the block
        out.free()
    with pytest.raises(backend.GpuBackendError, match="outside"):
        backend.Block.concat_pieces([(blocks[2], 30, 2)])
    for b in blocks:
        b.free()


def test_utf8_rewrite_at_tile_boundaries(gpu):
    """Invalid strings where the statistics' 1024-row tiles meet, in a column that is otherwise ASCII; NULs kept."""
    vals = [b"ab\0c"] * 5000
    for r in (0, 1023, 1024, 2047, 2048, 4999):
        vals[r] = b"x\xe4\xb8" if r % 2 else b"\xff\0\x80"
    offs = np.zeros(len(vals) + 1, np.uint32)
    np.cumsum([len(v) for v in vals], out=offs[1:])
    col = Column(T_STR, np.frombuffer(b"".join(vals), np.uint8).copy(), offs)
    b = backend.Block.upload(0, [col], len(vals))
    assert b.stats() == ([0], [6])
    out = backend.Block.concat_pieces([(b, 1000, 3000), (b, 4000, 1000)], [backend.CONCAT_UTF8])
    got = out.column(0, T_STR)
    want = [v.decode("utf-8", "replace").encode() for v in vals[1000:5000]]
    assert [got.data[got.offsets[i]:got.offsets[i + 1]].tobytes() for i in range(4000)] == want
    out.free()
    b.free()


# ---- pipelines against ref --------------------------------------------------------------------------------------------------
def _ref(ds):
    rows, names = ds._execute()
    return ds._ctx._dataset_from_rows(rows, names)


def _csv(ds, tmp_path, name):
    p = str(tmp_path / name)
    ds.tocsv(p, null_value="NA")
    return open(p, "rb").read()


def _same(a, b, tmp_path, tag=""):
    """a and b behave alike: rows, columns, types, cost, exception counts, tocsv bytes."""
    assert a.collect() == b.collect(), tag
    assert a.columns == b.columns and a.types == b.types and a._cost() == b._cost(), tag
    assert a.exception_counts == b.exception_counts, tag
    assert _csv(a, tmp_path, "a.csv") == _csv(b, tmp_path, "b.csv"), tag


def _f64_bits(v):
    return np.float64(v).view(np.int64).item()


def _downstream(ds):
    """Pipelines over a dataset of columns (k: int, s: Option[str], x: f64, n: Option[int])."""
    return {
        "map": ds.map(lambda r: (r["k"] * 3, r["s"] if r["s"] is not None else "-", r["x"] + 1.0)),
        "filter": ds.filter(lambda r: r["k"] % 3 != 0),
        "raises": ds.withColumn("q", lambda r: 100 // (r["k"] % 7)),
        "aggregate": ds.aggregate(lambda a, b: a + b, lambda a, r: a + r["x"] * 1.000001, 0.0),
        "byKey": ds.map(lambda r: (r["k"] % 5, r["x"])).aggregateByKey(lambda a, b: a + b, lambda a, r: a + r[1], 0.0, [0]),
        "unique": ds.map(lambda r: r["k"] % 11).unique(),
        "nonecol": ds.map(lambda r: (r["k"], r["n"] is None)),
    }


def _table(n, seed=1, all_none=True):
    rng = random.Random(seed)
    return [(i, None if i % 4 == 0 else "s%dé" % i, rng.uniform(-1e6, 1e6), None if all_none else i) for i in range(n)]


def _compare_pipelines(ctx, cached, ref, tmp_path):
    """The same operators (same ids, so exception counts compare key by key) over the cache and over ref."""
    for name, a in _downstream(cached).items():
        b = dataset.DataSet(ctx, ref._source, a._ops)
        ra, rb = a.collect(), b.collect()
        if name == "aggregate":
            assert [_f64_bits(v) for v in ra] == [_f64_bits(v) for v in rb], name
        assert ra == rb, name
        assert a.exception_counts == b.exception_counts, name
        assert a.types == b.types and a.columns == b.columns, name
    _same(cached, ref, tmp_path)


@pytest.mark.parametrize("n", [1, 33, 1000])
def test_row_stage_cache_equals_host_rows(gpu, tmp_path, n):
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 64})
    base = ctx.parallelize(_table(n), columns=["k", "s", "x", "n"]).filter(lambda r: r["k"] >= 0)
    before = ctx.metrics.cache_rows
    cached = base.cache()
    assert ctx.metrics.cache_rows - before == n
    assert isinstance(cached._source, dataset.CacheSource)
    ref = _ref(base)
    assert not isinstance(ref._source, dataset.CacheSource)
    assert [len(p.block.column_bytes()) for p in cached._source.rows.parts]  # blocks exist
    assert [int(p.info.n_out_rows) for p in cached._source.rows.parts] == [min(64, n - k) for k in range(0, n, 64)]
    assert cached._source.col_types == [c.type for c in ref._source.cols]
    assert cached._source.option_cols == ref._source.option_cols
    _compare_pipelines(ctx, cached, ref, tmp_path)


def test_invalid_utf8_and_reblocking_across_parts(gpu, tmp_path):
    """A byte slice through multi-byte characters leaves invalid UTF-8; a filter leaves stage results of different sizes, which
    are re-cut at blockRows."""
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 64})
    rows = [(i, "中éa" * (i % 4)) for i in range(700)]
    base = ctx.parallelize(rows, columns=["k", "s"]).filter(lambda r: r["k"] % 7 != 3).withColumn("cut", lambda r: r["s"][:4])
    cached = base.cache()
    ref = _ref(base)
    assert ctx.metrics.cache_rows == 600
    assert cached.collect() == ref.collect()
    assert cached.map(lambda r: (r["cut"], len(r["cut"]))).collect() == ref.map(lambda r: (r["cut"], len(r["cut"]))).collect()
    assert _csv(cached, tmp_path, "a.csv") == _csv(ref, tmp_path, "b.csv")
    assert [int(p.info.n_out_rows) for p in cached._source.rows.parts] == [64] * 9 + [24]


def test_reuse_branches_self_join_and_cache_of_cache(gpu, tmp_path):
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 64})
    base = ctx.parallelize(_table(300, all_none=False), columns=["k", "s", "x", "n"]).withColumn("m", lambda r: r["k"] % 10)
    cached = base.cache()
    ref = _ref(base)
    a, b = cached.filter(lambda r: r["m"] < 5), cached.map(lambda r: (r["k"], r["m"]))
    for _ in range(2):
        assert a.collect() == ref.filter(lambda r: r["m"] < 5).collect()
        assert b.collect() == ref.map(lambda r: (r["k"], r["m"])).collect()
    h = ctx.metrics.device_handoff_rows
    sj = cached.join(cached, "k", "k")
    assert sj.collect() == ref.join(ref, "k", "k").collect()
    assert ctx.metrics.device_handoff_rows - h >= 600  # both sides read the cache on the device
    assert cached.join(ref, "m", "m").collect() == ref.join(ref, "m", "m").collect()
    assert cached.leftJoin(ctx.parallelize([(1, "a"), (2, "b")], columns=["m", "t"]), "m", "m").collect() == \
        ref.leftJoin(ctx.parallelize([(1, "a"), (2, "b")], columns=["m", "t"]), "m", "m").collect()
    cc = cached.cache()
    assert cc._source is cached._source and ctx.metrics.cache_rows == 300
    _same(cc, ref, tmp_path)
    _same(cached, ref, tmp_path)


def test_cached_join_output(gpu, tmp_path):
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 64})
    L = ctx.parallelize([(i, "l%d" % i) for i in range(200)], columns=["k", "a"]).withColumn("b", lambda r: r["k"] * 2)
    R = ctx.parallelize([(i, "r%d" % i if i % 6 else None) for i in range(0, 300, 3)], columns=["k", "s"]).withColumn("t", lambda r: r["k"] + 1)
    for j in (L.join(R, "k", "k"), L.leftJoin(R, "k", "k")):
        before = ctx.metrics.cache_rows
        cached = j.cache()
        ref = _ref(j)
        assert ctx.metrics.cache_rows - before == len(ref.collect())
        _same(cached, ref, tmp_path)
        assert cached.join(L, "k", "k").collect() == ref.join(L, "k", "k").collect()
        assert L.join(cached, "k", "k").collect() == L.join(ref, "k", "k").collect()


def test_lifetime_and_metrics(gpu):
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 64})
    base = ctx.parallelize(_table(500, all_none=False), columns=["k", "s", "x", "n"]).filter(lambda r: r["k"] > 0)
    cached = base.cache()
    src = cached._source
    nbytes = ctx.metrics.cache_bytes
    exact = sum(499 * 8 for _ in range(3)) + sum(len(s.encode()) for _, s, _, _ in _table(500)[1:] if s is not None) + 499 * 4 + \
        len(src.rows.parts) * 4 + sum((int(p.info.n_out_rows) + 31) // 32 * 4 for p in src.rows.parts)
    assert nbytes == exact  # values, string bytes + offsets, the bitmap of the one column with None
    branch = cached.map(lambda r: r["k"])
    del cached, src
    gc.collect()
    assert ctx.metrics.cache_bytes == nbytes  # a branch still refers to it
    assert branch.collect() == list(range(1, 500))
    del branch
    gc.collect()
    assert ctx.metrics.cache_bytes == 0 and ctx.metrics.cache_rows == 499


def test_nomem_takes_the_host_path(gpu, tmp_path, monkeypatch):
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 64})
    base = ctx.parallelize(_table(300), columns=["k", "s", "x", "n"]).filter(lambda r: r["k"] % 2 == 0)
    real, calls = backend.Block.concat_pieces, []

    def failing(pieces, flags=None):
        calls.append(1)
        if len(calls) == 2:
            err = backend.GpuBackendError("tplx_gpu_block_concat_pieces failed (-5): out of device memory")
            err.code = backend.E_NOMEM
            raise err
        return real(pieces, flags)
    monkeypatch.setattr(backend.Block, "concat_pieces", staticmethod(failing))
    cached = base.cache()
    monkeypatch.undo()
    assert len(calls) == 2 and not isinstance(cached._source, dataset.CacheSource)
    assert ctx.metrics.cache_rows == 0 and ctx.metrics.cache_bytes == 0
    assert any("cache()" in m for m in ctx._messages)
    _same(cached, _ref(base), tmp_path)


class _NoCompiler:
    def __init__(self, *args, **kwargs):
        raise frontend.UnsupportedUDF("every stage on the CPython path")


@pytest.mark.parametrize("cond", ["devices", "no_option", "fallback", "interpreter", "resolve_misfit", "aggregate", "zero_rows",
                                  "bad_csv_rows"])
def test_host_path_conditions(gpu, tmp_path, cond, monkeypatch):
    conf = {"devices": {"tuplex.gpu.devices": "0,0"}, "no_option": {"tuplex.gpu.optionColumns": "false"}}.get(cond, {})
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 64, **conf})
    rows = [(i, "v%d" % i) for i in range(100)]
    if cond == "fallback":
        rows.append(("x", 1))
    if cond == "no_option":
        rows[5] = (5, None)
    if cond == "interpreter":
        monkeypatch.setattr(dataset, "StageCompiler", _NoCompiler)
    ds = ctx.parallelize(rows, columns=["k", "a"]).withColumn("c", lambda r: r["a"] + "!")
    if cond == "resolve_misfit":
        ds = ds.withColumn("q", lambda r: 10 // (r["k"] % 3)).resolve(ZeroDivisionError, lambda r: "zero")
    if cond == "aggregate":
        ds = ds.map(lambda r: (r["k"] % 4, r["k"])).aggregateByKey(lambda a, b: a + b, lambda a, r: a + r[1], 0, [0])
    if cond == "zero_rows":
        ds = ds.map(lambda r: r["k"]).filter(lambda k: k < 0)
    if cond == "bad_csv_rows":
        p = tmp_path / "bad.csv"
        p.write_text("k,a\n" + "".join("%d,v%d\n" % (i, i) for i in range(50)) + "7,x,extra\n")
        ds = ctx.csv(str(p)).withColumn("c", lambda r: r["a"] + "!")
    cached = ds.cache()
    assert ctx.metrics.cache_rows == 0
    assert not isinstance(cached._source, dataset.CacheSource)
    ref = _ref(ds)
    assert cached.collect() == ref.collect() and cached.columns == ref.columns and cached._cost() == ref._cost()
    if cond == "zero_rows":
        assert cached.collect() == [] and len(cached._source.cols) == 1 and cached._source.cols[0].type == T_I64


# ---- the reference's pipelines with their goldens ------------------------------------------------------------------------------
def test_zillow_z1_preload(gpu, tmp_path):
    src = tmp_path / "zillow.csv"
    src.write_bytes(gzip.open(os.path.join(workloads.GOLDEN, "zillow_noexc.csv.gz"), "rb").read())
    ctx = tuplex_b200.Context()
    ds = ctx.csv(str(src)).cache()
    assert ctx.metrics.cache_rows == 32661
    for k in range(2):
        workloads.zillow_pipeline(ds).tocsv(str(tmp_path / ("out%d" % k)))
        assert hashlib.md5((tmp_path / ("out%d" % k) / "part0.csv").read_bytes()).hexdigest() == "4d5ca0263b1a5058341a369116dee83a"
    assert workloads.zillow_pipeline(ds).types == workloads.zillow_pipeline(_ref(ctx.csv(str(src)))).types


def test_logs_io_shape(gpu, tmp_path):
    """runtuplex-io.py's shape: the text file and the blacklist cached, then the regex-free parse and the join."""
    from logs_udfs import ParseWithStrip
    logs, ips = _golden(tmp_path, "logs.sample.txt"), _golden(tmp_path, "bad_ips_all.txt")
    ctx = tuplex_b200.Context()
    text, bad = ctx.text(logs).cache(), ctx.csv(ips).cache()
    n_lines = ctx.metrics.cache_rows
    assert n_lines > 3437
    rows = text.map(ParseWithStrip).join(bad, "ip", "BadIPs").collect()
    assert len(rows) == 3437
    assert rows == ctx.text(logs).map(ParseWithStrip).join(ctx.csv(ips), "ip", "BadIPs").collect()
    blk = _golden(tmp_path, "ip_blacklist.csv")
    out = str(tmp_path / "logs.csv")
    text.map(ParseWithStrip).join(ctx.csv(blk).cache(), "ip", "BadIPs").selectColumns(["ip", "endpoint"]).tocsv(out)
    assert open(out, "rb").read() == b"ip,endpoint\n1.1.209.108,/research/finance/\n"


def test_311_weld_mode(gpu, tmp_path):
    from test_gpu_csv_option import NULLS_311, _cpython_311, fix_zip_codes, golden
    data = golden("311-service-requests-sf=1.csv")
    path = tmp_path / "sf1.csv"
    path.write_bytes(data)
    ctx = tuplex_b200.Context()
    ds = ctx.csv(str(path), null_values=NULLS_311, type_hints={0: typing.Optional[str]}).cache()
    assert ctx.metrics.cache_rows > 0
    got = ds.mapColumn("Incident Zip", fix_zip_codes).unique().collect()
    want = _cpython_311(data, NULLS_311)
    assert set(got) == want and len(got) == len(want)


def test_flights_like_simulate_spark_caches(gpu):
    import test_flights_like as fl
    flights, carriers, airports = fl._tables(3000, 5)
    want, want_names = fl._expected(flights, carriers, airports)
    c = tuplex_b200.Context({"tuplex.gpu.blockRows": 700})
    df = c.parallelize(flights, columns=fl.F_COLS).cache()
    df = df.withColumn('OriginCity', lambda x: x['OriginCityName'][:x['OriginCityName'].rfind(',')].strip())
    df = df.withColumn('OriginState', lambda x: x['OriginCityName'][x['OriginCityName'].rfind(',') + 1:].strip())
    df = df.withColumn('DestCity', lambda x: x['DestCityName'][:x['DestCityName'].rfind(',')].strip())
    df = df.mapColumn('CrsArrTime', lambda x: '{:02}:{:02}'.format(int(x / 100), x % 100) if x else None)
    df = df.withColumn('CancellationCode', fl.cleanCode)
    df = df.mapColumn('Diverted', lambda x: True if x > 0 else False)
    df = df.withColumn('CancellationReason', fl.divertedUDF)
    df = df.withColumn('ActualElapsedTime', fl.fillInTimesUDF).ignore(TypeError).cache()
    dc = c.parallelize(carriers, columns=fl.C_COLS)
    dc = dc.withColumn('AirlineName', lambda x: x['Description'][:x['Description'].rfind('(')].strip())
    dc = dc.withColumn('AirlineYearFounded', lambda x: int(x['Description'][x['Description'].rfind('(') + 1:x['Description'].rfind('-')]))
    dc = dc.withColumn('AirlineYearDefunct', fl.extractDefunctYear).cache()
    da = c.parallelize(airports, columns=fl.A_COLS).cache()
    dall = df.join(dc, 'OpUniqueCarrier', 'Code').cache()
    dall = dall.leftJoin(da, 'Origin', 'IATACode', prefixes=(None, 'Origin'))
    dall = dall.leftJoin(da, 'Dest', 'IATACode', prefixes=(None, 'Dest')).cache()
    dall = dall.mapColumn('Distance', lambda x: x / 0.00062137119224)
    dall = dall.mapColumn('AirlineName', lambda s: s.replace('Inc.', '').replace('LLC', '').replace('Co.', '').strip())
    dall = dall.renameColumn('AirlineName', 'CarrierName').renameColumn('Origin', 'OriginAirportIATACode')
    dall = dall.filter(fl.filterDefunctFlights)
    assert dall.columns == want_names
    assert dall.collect() == want
    assert c.metrics.cache_rows > len(flights)
