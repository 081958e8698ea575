"""The device key sort (K11, tplx_gpu_result_sort_by_keys) against Python's stable sorted(), and aggregateByKey / unique() results
that stay on the device: the next stage, a join and tocsv take the sorted groups there, collect() fetches them in device order. Every
pipeline is checked against a plain Python reference computed from the input rows, and ctx.metrics.device_handoff_rows shows which
path ran; the host-path conditions give the same rows with no handoff."""
import os
import random
import struct
import typing

import numpy as np
import pytest

import tuplex_b200
from tuplex_b200 import backend, dataset, frontend
from tuplex_b200.backend import Column, pack_valid
from tuplex_b200.ir import C, T_BOOL, T_F64, T_I64, T_STR

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


# ---- tplx_gpu_result_sort_by_keys ---------------------------------------------------------------------------------------------
def _stage_result(cols, option=()):
    """A stage result holding `cols` (identity stage; Option columns keep their bitmaps)."""
    names = ["c%d" % i for i in range(len(cols))]
    sc = frontend.StageCompiler([c.type for c in cols], names, list(option))
    st = backend.Stage(sc.finish_memory())
    n = len(cols[0])
    res = st.run_host(0, cols, n)
    assert int(res.info.n_out_rows) == n and int(res.info.n_exceptions) == 0
    return res


def _order(vals, nk):
    """Python's stable sort of the row indices by the first nk columns, None first."""
    def key(i):
        return tuple((0,) if vals[c][i] is None else (1, vals[c][i]) for c in range(nk))
    return sorted(range(len(vals[0])), key=key)


def _values(col):
    """Python values of a column, f64 values as their bits (NaN payloads and -0.0 compare exactly)."""
    vals = col.to_values()
    return [struct.pack("<d", v) if isinstance(v, float) else v for v in vals]


def _check_sorted(cols, nk, option=(), flags=None):
    res = _stage_result(cols, option)
    vals = [_values(c) for c in cols]
    out = res.sort_by_keys(nk, flags)
    perm = _order(vals, nk)
    assert int(out.info.n_out_rows) == len(perm) and int(out.info.n_exceptions) == 0
    assert out.info.kernel_launches >= len(cols)
    for c, g in enumerate(out.columns()):
        assert _values(g) == [vals[c][i] for i in perm], c
        dropped = flags is not None and flags[c] & backend.CONCAT_DROP_VALID
        assert (g.valid is None) == bool(dropped or c not in option), c
    assert [_values(c) for c in res.columns()] == vals  # the input result is unchanged
    out.free()
    res.free()


def _opt(col, present):
    return Column(col.type, col.data, col.offsets, pack_valid(present))


I64_EDGES = [-(1 << 63), (1 << 63) - 1, 0, -1, 1, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, -(1 << 32) - 1, -(1 << 32) + 1]


@pytest.mark.parametrize("n", [0, 1, 4095, 4096, 4097, (1 << 21) + 1])
def test_i64_keys(gpu, n):
    rng = np.random.default_rng(n)
    k = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64)
    edge = rng.random(n) < 0.3
    k[edge] = np.array(I64_EDGES, np.int64)[rng.integers(0, len(I64_EDGES), int(edge.sum()))]
    payload = Column(T_I64, np.arange(n, dtype=np.int64))
    _check_sorted([Column(T_I64, k), payload], 1)


def test_bool_and_small_ranges(gpu):
    rng = np.random.default_rng(1)
    n = 9000
    b = Column(T_BOOL, rng.integers(0, 2, n).astype(np.int64))
    small = Column(T_I64, rng.integers(-3, 300, n).astype(np.int64))  # two digits vary, the rest are skipped
    _check_sorted([b, small, Column(T_I64, np.arange(n, dtype=np.int64))], 2)
    _check_sorted([small, b], 1)


@pytest.mark.parametrize("t", [T_I64, T_STR, T_BOOL], ids=["i64", "str", "bool"])
def test_option_keys_none_first(gpu, t):
    rng = np.random.default_rng(t)
    n = 5000
    if t == T_STR:
        base = Column.from_values(["".join(rng.choice(list("ab\0é"), rng.integers(0, 12))) for _ in range(n)], T_STR)
    elif t == T_BOOL:
        base = Column(T_BOOL, rng.integers(0, 2, n).astype(np.int64))
    else:
        base = Column(T_I64, rng.integers(-5, 5, n).astype(np.int64))
    key = _opt(base, rng.random(n) >= 0.2)
    _check_sorted([key, Column(T_I64, np.arange(n, dtype=np.int64))], 1, option=[0])


def _str_col(strs):
    return Column.from_values(strs, T_STR)


def test_string_edges(gpu):
    strs = ["", "", "a\0", "a", "ab", "a\0\0", "\0", "", "\0\0", "é", "ÿ", "€", "𝄞", "a" * 8, "a" * 8 + "\0", "a" * 9, "a" * 7 + "\0"]
    strs = strs * 3
    random.Random(2).shuffle(strs)
    _check_sorted([_str_col(strs), Column(T_I64, np.arange(len(strs), dtype=np.int64))], 1)
    assert sorted(["a", "a\0", "a\0\0", "ab"]) == ["a", "a\0", "a\0\0", "ab"]


def test_string_lengths_0_to_257(gpu):
    """Lengths 0-257 over a 2-letter alphabet (long shared prefixes, many rounds and skips); string starts at every offset mod 16."""
    rng = random.Random(4)
    strs = ["".join(rng.choice("ab") for _ in range(rng.randrange(0, 258))) for _ in range(3000)]
    strs += ["a" * n for n in range(258)] + ["a" * n + "b" for n in range(0, 258, 7)]
    rng.shuffle(strs)
    offs = np.cumsum([0] + [len(s) for s in strs]) % 16
    assert set(offs.tolist()) == set(range(16))
    _check_sorted([_str_col(strs), Column(T_I64, np.arange(len(strs), dtype=np.int64))], 1)


def test_strings_sharing_a_1mib_prefix(gpu):
    rng = random.Random(5)
    prefix = "".join(rng.choice("xyz") for _ in range(1 << 20))
    strs = [prefix + chr(0x41 + i) for i in range(64)]
    rng.shuffle(strs)
    _check_sorted([_str_col(strs), Column(T_I64, np.arange(64, dtype=np.int64))], 1)


@pytest.mark.parametrize("n", [4097, (1 << 21) + 1])
def test_string_keys_large(gpu, n):
    rng = np.random.default_rng(n)
    ids = rng.integers(0, n // 3, n)
    strs = ["k%d" % i + "x" * (i % 9) for i in ids.tolist()]
    _check_sorted([_str_col(strs), Column(T_I64, np.arange(n, dtype=np.int64))], 1)


F64_EDGES = [struct.unpack("<d", struct.pack("<Q", b))[0] for b in
             (0x7FF8000000000123, 0xFFF0000000000001, 0x8000000000000000, 0x7FF0000000000000, 0x0000000000000001)]


def test_two_and_max_keys_with_payloads(gpu):
    rng = np.random.default_rng(9)
    n = 20000
    s = _str_col(["".join(rng.choice(list("abc"), rng.integers(0, 4))) for _ in range(n)])
    i = Column(T_I64, rng.integers(-2, 2, n).astype(np.int64))
    b = Column(T_BOOL, rng.integers(0, 2, n).astype(np.int64))
    f = rng.standard_normal(n)
    edge = rng.random(n) < 0.3
    f[edge] = np.array(F64_EDGES)[rng.integers(0, len(F64_EDGES), int(edge.sum()))]
    pay = Column(T_F64, f)
    os_ = _opt(_str_col(["p%d" % k for k in range(n)]), rng.random(n) >= 0.5)
    oi = _opt(Column(T_I64, rng.integers(0, 3, n).astype(np.int64)), rng.random(n) >= 0.3)
    full = _opt(Column(T_I64, np.arange(n, dtype=np.int64)), np.ones(n, bool))  # a bitmap without None: DROP_VALID drops it
    _check_sorted([s, i, pay, os_, full], 2, option=[3, 4])
    _check_sorted([s, i, pay, os_, full], 2, option=[3, 4], flags=[0, 0, 0, 0, backend.CONCAT_DROP_VALID])
    nk = C["TPLX_MAX_KEYS"]
    cols = [oi, s, b, i, s, oi, b, i, pay, os_]
    assert len(cols) >= nk + 1
    _check_sorted(cols, nk, option=[0, 5, 9])


def test_stable_with_duplicate_keys(gpu):
    rng = np.random.default_rng(11)
    n = 30000
    k = Column(T_I64, rng.integers(0, 7, n).astype(np.int64))
    s = _str_col([["x", "y", "xy"][v] for v in rng.integers(0, 3, n).tolist()])
    _check_sorted([k, s, Column(T_I64, np.arange(n, dtype=np.int64))], 2)
    _check_sorted([s, Column(T_I64, np.arange(n, dtype=np.int64))], 1)


def test_error_codes(gpu):
    res = _stage_result([Column(T_I64, np.arange(10, dtype=np.int64)), Column(T_F64, np.zeros(10))])
    for nk, flags in [(0, None), (C["TPLX_MAX_KEYS"] + 1, None), (3, None), (1, [4, 0]), (1, [2, 0])]:
        with pytest.raises(backend.GpuBackendError) as e:
            res.sort_by_keys(nk, flags)
        assert e.value.code == -4, (nk, flags)  # TPLX_E_BADARG
    with pytest.raises(backend.GpuBackendError) as e:
        res.sort_by_keys(2)
    assert e.value.code == -6  # TPLX_E_UNSUPPORTED: f64 key
    res.free()


# ---- through Context --------------------------------------------------------------------------------------------------------
def _rows(n, seed=0):
    rng = random.Random(seed)
    words = ["", "a", "ab", "b", "é", "k\0", "zz", "x" * 20, "x" * 20 + "y"]
    return [(rng.choice(words) + str(rng.randrange(n // 4 + 1)), rng.randrange(-50, 50)) for _ in range(n)]


def _groups(rows, key, val, order=lambda k: (k is not None, k)):
    """aggregateByKey(sum) in Python: groups ordered by key, None first."""
    table = {}
    for r in rows:
        table[key(r)] = table.get(key(r), 0) + val(r)
    return sorted(table.items(), key=lambda kv: order(kv[0]))


@pytest.fixture
def no_host_sort(monkeypatch):
    def boom(k):
        raise AssertionError("the host path sorted the groups")
    monkeypatch.setattr(dataset, "_key_order", boom)


def _by_key(ds):
    return ds.aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["k"])


def test_aggregate_by_key_and_unique_collect(gpu, no_host_sort):
    rows = _rows(5000)
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 700})
    ds = ctx.parallelize(rows, columns=["k", "v"])
    assert _by_key(ds).collect() == _groups(rows, lambda r: r[0], lambda r: r[1])
    assert ds.map(lambda x: x["k"]).unique().collect() == sorted({r[0] for r in rows})
    assert ds.unique().collect() == sorted(set(rows))
    assert ctx.metrics.device_handoff_rows == 0  # collect does not count


def test_next_stage_and_tocsv(gpu, no_host_sort, tmp_path):
    rows = _rows(6000, 1)
    want = _groups(rows, lambda r: r[0], lambda r: r[1])
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 500})
    g = _by_key(ctx.parallelize(rows, columns=["k", "v"]))
    h0 = ctx.metrics.device_handoff_rows
    got = g.map(lambda x: (x[0] + "!", x[1] * 2)).filter(lambda x: x[1] != 0).collect()
    assert got == [(k + "!", v * 2) for k, v in want if v != 0]
    assert ctx.metrics.device_handoff_rows - h0 == len(want)
    h0 = ctx.metrics.device_handoff_rows
    got = g.withColumn("n", lambda x: x[1] - 1).collect()
    assert got == [(k, v, v - 1) for k, v in want]
    assert ctx.metrics.device_handoff_rows - h0 == len(want)
    h0 = ctx.metrics.device_handoff_rows
    out = str(tmp_path / "g.csv")
    g.tocsv(out, header=False)
    assert open(out, "rb").read() == "".join("%s,%d\n" % (dataset._csv_cell(k), v) for k, v in want).encode()
    assert ctx.metrics.device_handoff_rows - h0 == len(want)
    h0 = ctx.metrics.device_handoff_rows
    out = str(tmp_path / "m.csv")
    g.map(lambda x: (x[1], x[0])).tocsv(out, header=False)
    assert open(out, "rb").read() == "".join("%d,%s\n" % (v, dataset._csv_cell(k)) for k, v in want).encode()
    assert ctx.metrics.device_handoff_rows - h0 == len(want)


def test_group_by_then_group_by(gpu, no_host_sort):
    rows = _rows(4000, 2)
    want = _groups(rows, lambda r: r[0], lambda r: r[1])
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 300})
    g = _by_key(ctx.parallelize(rows, columns=["k", "v"]))
    got = g.map(lambda x: (x[1] % 5, x[1])).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x[1], 0, [0]).collect()
    assert got == _groups(want, lambda r: r[1] % 5, lambda r: r[1])
    assert ctx.metrics.device_handoff_rows == len(want)


def test_f64_aggregate_after_group_by_same_bits(gpu):
    rng = random.Random(3)
    # group sums are exact (quarters), so only the cut of the groups into blocks can change the f64 aggregate's bits
    rows = [("g%d" % rng.randrange(3000), rng.randrange(-1600, 1600) * 0.25) for _ in range(20000)]
    res = {}
    for conf in ({}, {"tuplex.gpu.devices": "0,0"}):
        ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 256, **conf})
        g = ctx.parallelize(rows, columns=["k", "v"]).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0.0, ["k"])
        total = g.aggregate(lambda a, b: a + b, lambda a, x: a + x[1] * 0.1, 0.0).collect()
        res[bool(conf)] = (struct.pack("<d", total[0]), ctx.metrics.device_handoff_rows)
    groups = {r[0] for r in rows}
    assert len(groups) > 256
    assert res[False][0] == res[True][0]
    assert res[False][1] == len(groups) and res[True][1] == 0


@pytest.mark.parametrize("kind", ["inner", "left"])
@pytest.mark.parametrize("groups_left", [True, False], ids=["groups_left", "groups_right"])
def test_join_sides(gpu, no_host_sort, kind, groups_left):
    rows = _rows(3000, 4)
    want = _groups(rows, lambda r: r[0], lambda r: r[1])
    rng = random.Random(8)
    other_rows = [(k, rng.randrange(100)) for k, _ in want if rng.random() < 0.6] + [("nope", 1), ("", 2)]
    ctx = tuplex_b200.Context()
    g = _by_key(ctx.parallelize(rows, columns=["k", "v"]))
    other = ctx.parallelize(other_rows, columns=["k2", "w"])
    ds = (g.join if kind == "inner" else g.leftJoin) if groups_left else (other.join if kind == "inner" else other.leftJoin)
    got = ds(other, "k", "k2").collect() if groups_left else ds(g, "k2", "k").collect()
    L, R = (want, other_rows) if groups_left else (other_rows, want)
    ref = dataset._py_join_pairs([tuple(r) for r in L], 0, [tuple(r) for r in R], 0, kind == "left", True, 2)
    assert sorted(got, key=repr) == sorted(ref, key=repr)
    assert ctx.metrics.device_handoff_rows >= len(want)


def test_311_unique_tocsv(gpu, tmp_path, no_host_sort):
    from test_gpu_csv_option import NULLS_311, _cpython_311, fix_zip_codes, golden
    data = golden("311-service-requests-sf=1.csv")
    path = tmp_path / "sf1.csv"
    path.write_bytes(data)
    want = _cpython_311(data, NULLS_311)
    ctx = tuplex_b200.Context()
    out = str(tmp_path / "out")
    ctx.csv(str(path), null_values=NULLS_311, type_hints={0: typing.Optional[str]}).mapColumn("Incident Zip", fix_zip_codes).unique().tocsv(out)
    txt = open(os.path.join(out, "part0.csv"), "rb").read().decode()
    ordered = sorted(want, key=lambda v: (v is not None, v or ""))
    assert txt.split("\n") == ["Incident Zip"] + [dataset._csv_cell(v) for v in ordered] + [""]
    assert len(want) == 246 and ctx.metrics.device_handoff_rows == 246


# ---- host-path conditions -------------------------------------------------------------------------------------------------------
def _python_by_key_map(rows, key, val):
    return [(k, v + 1) for k, v in _groups(rows, key, val)]


@pytest.mark.parametrize("cond", ["devices", "no_option", "raises", "fallback", "cut_utf8", "all_none", "zero_groups"])
def test_host_path_conditions(gpu, cond, tmp_path):
    conf = {"devices": {"tuplex.gpu.devices": "0,0"}, "no_option": {"tuplex.gpu.optionColumns": "false"}}.get(cond, {})
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 400, **conf})
    rows = [("é%d" % (i % 37), i) for i in range(1000)]
    if cond == "fallback":
        rows.append((5, 5))
    ds = ctx.parallelize(rows, columns=["k", "v"])
    key, val = (lambda r: r[0]), (lambda r: r[1])
    if cond == "raises":
        ds = ds.mapColumn("v", lambda v: 100 // (v % 7))
        val = lambda r: 100 // (r[1] % 7)  # noqa: E731
        rows = [r for r in rows if r[1] % 7]  # the rows that raise are dropped
    if cond == "cut_utf8":
        ds = ds.mapColumn("k", lambda k: k[:1])  # byte slice: half of "é"
        key = lambda r: "�"  # noqa: E731
    if cond == "all_none":
        ds = ds.mapColumn("k", lambda k: None if len(k) > 0 else k)
        key = lambda r: None  # noqa: E731
    if cond == "zero_groups":
        ds = ds.filter(lambda r: r["v"] < 0)
    if cond == "fallback":
        key = lambda r: r[0]  # noqa: E731
    g = ds.aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["k"])
    if cond == "zero_groups":  # tocsv: a stage after zero groups has no rows to type its source from
        out = str(tmp_path / "z.csv")
        g.tocsv(out, header=False)
        assert open(out, "rb").read() == b"" and ctx.metrics.device_handoff_rows == 0
        return
    got = g.map(lambda x: (x[0], x[1] + 1)).collect()
    if cond == "fallback":
        want = [(k, v + 1) for k, v in _groups(rows, key, val, order=lambda k: dataset._key_order((k,)))]
    else:
        want = _python_by_key_map(rows, key, val)
    assert got == want
    assert ctx.metrics.device_handoff_rows == 0


def test_option_key_without_none(gpu, tmp_path):
    """A key column typed Option[str] that holds no None: the groups lose the bitmap as the host path's rows would, so the next
    stage, types and tocsv match the host path."""
    rows = [("k%d" % (i % 50), i) for i in range(2000)]
    outs = {}
    for conf in ({}, {"tuplex.gpu.devices": "0,0"}):
        ctx = tuplex_b200.Context(conf)
        g = ctx.parallelize(rows, columns=["k", "v"]).mapColumn("k", lambda k: None if k == "never" else k) \
            .aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["k"])
        nxt = g.map(lambda x: (x[0] + "?", x[1]))
        out = str(tmp_path / ("o%d.csv" % len(conf)))
        nxt.tocsv(out)
        outs[bool(conf)] = (nxt.collect(), nxt.types, g.types, open(out, "rb").read(), ctx.metrics.device_handoff_rows)
    dev, host = outs[False], outs[True]
    assert dev[:4] == host[:4]
    assert dev[4] > 0 and host[4] == 0
