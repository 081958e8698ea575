"""Stages split at the operators the device cannot compile, on the GPU: every pipeline runs split (device segments around the CPython
operator) and as one CPython stage, and both are compared with a plain-Python evaluation written here: rows in order, exception
counts, columns, types and CSV bytes. tplx_gpu_block_select is checked against numpy on every column type at its size edges.
CPU twin: tests/test_stage_split.py (read sets, planning, column typing)."""
import gzip
import os
import random
import re
import string
from collections import Counter

import numpy as np
import pytest

import tuplex_b200 as tuplex
from tuplex_b200 import backend, dataset, pyexec
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR
from tuplex_b200.textsource import read_lines
from logs_udfs import ParseWithStrip

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = ["a", "s", "f"]
WORDS = ["alpha beta", "gamma", "delta epsilon zeta", "eta theta", "iota", "kappa lambda", "", "mu nu xi"]


def make_rows(n=3000, seed=7):
    r = random.Random(seed)
    return [(r.randrange(-50, 1000), r.choice(WORDS), round(r.uniform(-100, 100), r.randrange(1, 6))) for _ in range(n)]


# ---- plain Python evaluation of a pipeline: [("map" | "filter" | "withColumn" | "mapColumn", column, udf, resolvers, ignores)] ----
def step(kind, udf, column=None, resolve=(), ignore=()):
    return (kind, column, udf, list(resolve), list(ignore))


def py_eval(rows, names, steps):
    out, counts = [], Counter()
    for row in rows:
        vals, nm = list(row if isinstance(row, tuple) else (row,)), list(names)
        for kind, column, udf, resolvers, ignores in steps:
            d = dict(zip(nm, vals))

            def call(f):
                if kind == "mapColumn":
                    return f(d[column])
                return f(d if len(vals) > 1 else vals[0])
            try:
                try:
                    res = call(udf)
                except Exception as e:
                    if any(isinstance(e, c) for c in ignores):
                        vals = None
                        break
                    res = next((call(f) for c, f in resolvers if isinstance(e, c)), e)
                    if res is e:
                        raise
            except Exception as e:
                counts[(kind, type(e).__name__)] += 1
                vals = None
                break
            if kind == "filter":
                if not res:
                    vals = None
                    break
            elif kind == "map":
                vals, nm = list(res.values()), list(res.keys())
            elif column in nm:
                vals[nm.index(column)] = res
            else:
                vals, nm = vals + [res], nm + [column]
        if vals is not None:
            out.append(tuple(vals) if len(vals) > 1 else vals[0])
    return out, counts


def build(ds, steps):
    for kind, column, udf, resolvers, ignores in steps:
        ds = {"map": lambda: ds.map(udf), "filter": lambda: ds.filter(udf), "withColumn": lambda: ds.withColumn(column, udf),
              "mapColumn": lambda: ds.mapColumn(column, udf)}[kind]()
        for c, f in resolvers:
            ds = ds.resolve(c, f)
        for c in ignores:
            ds = ds.ignore(c)
    return ds


def by_kind(ds, counts):
    """exception_counts (keyed by operator id relative to the first operator) keyed by operator kind, as py_eval keys them."""
    kinds = {op.id - ds._ops[0].id: op.kind for op in ds._ops}
    out = Counter()
    for (op_id, name), k in counts.items():
        out[(kinds.get(op_id, "?"), name)] += k
    return out


def run_both(monkeypatch, make, action="collect", tmp_path=None, conf=None, unordered=False):
    """(split result, whole-stage result, split context): each result is (rows or CSV bytes, exception counts, columns, types)."""
    def once(ctx):
        first_id = pyexec.Op._next_id  # exception counts are keyed by operator id: count from the first operator of this build
        ds = make(ctx)
        if action == "tocsv":
            out = str(tmp_path / f"out{id(ctx)}.csv")
            ds.tocsv(out)
            got = open(out, "rb").read()
        else:
            got = ds.collect()
        counts = {(op - first_id, name): k for (op, name), k in ds.exception_counts.items()}
        metrics = (ctx.metrics.split_stages, ctx.metrics.interpreter_values)
        return got, counts, ds.columns, ds.types, ds, metrics  # (`types` runs the pipeline again over its first rows)
    split = once(tuplex.Context(conf or {}))
    with monkeypatch.context() as mp:
        mp.setattr(dataset, "_split_point", lambda *a, **k: None)
        whole = once(tuplex.Context(conf or {}))
        assert whole[5] == (0, 0)
    if unordered:  # unique(): the device orders its groups, the CPython path keeps them in first-seen order
        split, whole = (sorted(split[0], key=repr),) + split[1:], (sorted(whole[0], key=repr),) + whole[1:]
    assert split[:4] == whole[:4]
    return split, whole, split[5]


def check(monkeypatch, rows, names, steps, n_splits=1, columnwise=True, conf=None, tail=None, unordered=False):
    def make(ctx):
        ds = build(ctx.parallelize(rows, columns=names), steps)
        return tail(ds) if tail else ds
    split, _, (splits, values) = run_both(monkeypatch, make, conf=conf, unordered=unordered)
    if tail is None:
        want, counts = py_eval(rows, names, steps)
        assert split[0] == want
        assert by_kind(split[4], split[1]) == counts
    assert splits == n_splits
    assert (values > 0) == columnwise
    assert not any("falls back" in m for m in split[4]._ctx._messages)
    return split


CAP = step("mapColumn", lambda v: string.capwords(v), "s")
WORD1 = step("withColumn", lambda x: x["s"].split(" ")[1], "w")
ROUND = step("withColumn", lambda x: round(x["f"], 2), "r")
PCT = step("withColumn", lambda x: "%.2f" % x["f"], "p")
RESUB = step("mapColumn", lambda v: re.sub("[aeiou]", "_", v), "s")


@pytest.mark.parametrize("steps", [
    [CAP, step("withColumn", lambda x: len(x["s"]) + x["a"], "n"), step("filter", lambda x: x["n"] % 3 != 0)],
    [step("withColumn", lambda x: x["a"] * 2, "g"), step("withColumn", lambda x: x["s"].split(" ")[0], "w"),
     step("filter", lambda x: x["g"] % 3 != 0)],
    [step("filter", lambda x: x["a"] % 5 != 0), ROUND],
    [step("filter", lambda x: x["a"] > 100), PCT, step("withColumn", lambda x: x["p"] + "!", "q")],
    [step("withColumn", lambda x: x["a"] + 1, "b"), RESUB, step("mapColumn", lambda v: v.upper(), "s")],
], ids=["capwords_first", "split_middle", "round_last", "percent_format", "re_sub"])
def test_u_first_middle_last(gpu, monkeypatch, steps):
    check(monkeypatch, make_rows(), NAMES, steps)


@pytest.mark.parametrize("mode", ["raise", "resolve", "ignore"])
def test_u_that_raises(gpu, monkeypatch, mode):
    u = step("withColumn", lambda x: x["s"].split(" ")[1], "w", resolve=[(IndexError, lambda x: x["s"] + "?")] if mode == "resolve" else (),
             ignore=[IndexError] if mode == "ignore" else ())
    split = check(monkeypatch, make_rows(), NAMES, [step("withColumn", lambda x: 100 // (x["a"] % 7), "q"), u,
                                                    step("withColumn", lambda x: len(x["w"]), "n")])
    assert any(name == "ZeroDivisionError" for _, name in split[1])
    assert any(name == "IndexError" for _, name in split[1]) == (mode == "raise")


def test_unsupported_filter(gpu, monkeypatch):
    check(monkeypatch, make_rows(), NAMES, [step("withColumn", lambda x: str(x["a"]), "t"), step("filter", lambda x: x["t"].isdigit()),
                                            step("withColumn", lambda x: x["a"] * 3, "b")])


def test_two_unsupported_operators(gpu, monkeypatch):
    check(monkeypatch, make_rows(), NAMES, [step("filter", lambda x: x["a"] % 4 != 1), CAP, step("withColumn", lambda x: x["a"] - 1, "b"),
                                            ROUND, step("filter", lambda x: x["b"] > 0)], n_splits=2)


def test_option_result(gpu, monkeypatch):
    split = check(monkeypatch, make_rows(), NAMES, [
        step("filter", lambda x: x["a"] != 0), step("withColumn", lambda x: None if x["a"] % 3 == 0 else string.capwords(x["s"]), "o"),
        step("withColumn", lambda x: x["o"] is None, "none")])
    assert split[3][3] is not str  # typing.Optional[str]


@pytest.mark.parametrize("udf", [lambda x: round(x["f"]) if x["a"] % 2 else string.capwords(x["s"]),
                                 lambda x: None if x["s"].isdigit() else None,
                                 lambda x: round(x["f"]) * 10 ** 20 + x["a"]],
                         ids=["mixed_types", "all_none", "beyond_i64"])
def test_give_up_takes_the_row_path(gpu, monkeypatch, udf):
    check(monkeypatch, make_rows(500), NAMES, [step("filter", lambda x: x["a"] > 0), step("withColumn", udf, "g")], columnwise=False)


def test_map_takes_the_row_path(gpu, monkeypatch):
    check(monkeypatch, make_rows(), NAMES, [step("filter", lambda x: x["a"] > 0),
                                            step("map", lambda x: {"a": x["a"], "c": string.capwords(x["s"])}),
                                            step("withColumn", lambda x: x["a"] + len(x["c"]), "n")], columnwise=False)


def test_many_blocks(gpu, monkeypatch):
    check(monkeypatch, make_rows(5000), NAMES, [step("filter", lambda x: x["a"] % 3 != 0), CAP, step("filter", lambda x: len(x["s"]) > 4),
                                                WORD1], conf={"tuplex.gpu.blockRows": 700}, n_splits=2)


# ---- endpoints, joins, cache -------------------------------------------------------------------------------------------------------
PRE = [step("withColumn", lambda x: x["a"] % 10, "k"), CAP]


def test_before_aggregate(gpu, monkeypatch):
    split = check(monkeypatch, make_rows(), NAMES, PRE, tail=lambda ds: ds.aggregate(lambda a, b: a + b, lambda a, x: a + (x["k"] + len(x["s"])), 0))
    want, _ = py_eval(make_rows(), NAMES, PRE)
    assert split[0] == [sum(r[3] + len(r[1]) for r in want)]


def test_before_aggregate_by_key(gpu, monkeypatch):
    check(monkeypatch, make_rows(), NAMES, PRE + [step("filter", lambda x: x["a"] > 0)],
          tail=lambda ds: ds.aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["a"], 0, ["k"]))


def test_before_unique(gpu, monkeypatch):
    split = check(monkeypatch, make_rows(), NAMES, [step("filter", lambda x: x["a"] > 500), CAP],
                  tail=lambda ds: ds.selectColumns(["s"]).unique(), unordered=True)
    want, _ = py_eval(make_rows(), NAMES, [step("filter", lambda x: x["a"] > 500), CAP])
    assert sorted(split[0]) == sorted({r[1] for r in want})


def _right(ctx):
    return ctx.parallelize([(k, "k%d" % k) for k in range(0, 10)] + [(k, "x%d" % k) for k in range(0, 10, 3)], columns=["k", "label"])


def test_before_and_after_join(gpu, monkeypatch):
    rows = make_rows()
    check(monkeypatch, rows, NAMES, PRE, tail=lambda ds: ds.join(_right(ds._ctx), "k", "k"))
    check(monkeypatch, rows, NAMES, [step("withColumn", lambda x: x["a"] % 10, "k")], n_splits=1,
          tail=lambda ds: ds.join(_right(ds._ctx), "k", "k").withColumn("t", lambda x: x["label"] + "/").mapColumn(
              "s", lambda v: string.capwords(v)))


def test_before_cache(gpu, monkeypatch):
    rows = make_rows()
    split = check(monkeypatch, rows, NAMES, PRE, tail=lambda ds: ds.cache().filter(lambda x: x["k"] > 2))
    want, _ = py_eval(rows, NAMES, PRE)
    assert split[0] == [r for r in want if r[3] > 2]


# ---- file sources and the CSV sink ---------------------------------------------------------------------------------------------
def test_csv_source_and_sink(gpu, monkeypatch, tmp_path):
    rows = [r for r in make_rows(2000) if r[1]]  # an empty cell would be a null
    p = tmp_path / "in.csv"
    p.write_text("a,s,f\n" + "".join(f"{a},{s},{f!r}\n" for a, s, f in rows))

    def make(ctx):
        return build(ctx.csv(str(p)), [step("filter", lambda x: x["a"] % 3 != 0), CAP, step("withColumn", lambda x: x["a"] * 2, "b")])
    split, _, (splits, values) = run_both(monkeypatch, make, "tocsv", tmp_path)
    assert splits == 1 and values > 0 and split[4]._ctx.metrics.csv_rows > 0
    want, _ = py_eval(rows, NAMES, [step("filter", lambda x: x["a"] % 3 != 0), CAP, step("withColumn", lambda x: x["a"] * 2, "b")])
    assert split[0].decode().splitlines()[1:] == [",".join(dataset._csv_cell(v) for v in r) for r in want]


def test_u_last_to_csv(gpu, monkeypatch, tmp_path):
    rows = make_rows(2000)

    def make(ctx):
        return build(ctx.parallelize(rows, columns=NAMES), [step("filter", lambda x: x["a"] % 3 != 0), ROUND])
    split, _, (splits, values) = run_both(monkeypatch, make, "tocsv", tmp_path)
    want, _ = py_eval(rows, NAMES, [step("filter", lambda x: x["a"] % 3 != 0), ROUND])
    assert splits == 1 and values == len(want)
    assert split[0].decode().splitlines()[1:] == [",".join(dataset._csv_cell(v) for v in r) for r in want]


def test_text_source(gpu, monkeypatch, tmp_path):
    p = tmp_path / "in.txt"
    lines = [w + " " + str(i) for i, w in enumerate(WORDS * 300)]
    p.write_text("\n".join(lines) + "\n")

    def make(ctx):
        return ctx.text(str(p)).map(lambda x: {"line": x, "n": len(x)}).mapColumn("line", lambda v: string.capwords(v)).filter(
            lambda x: x["n"] > 6)
    split, _, (splits, values) = run_both(monkeypatch, make)
    assert split[0] == [(string.capwords(ln), len(ln)) for ln in lines if len(ln) > 6]
    assert splits == 1 and values == len(lines) and split[4]._ctx.metrics.text_rows >= len(lines)


def _golden(tmp_path, name):
    f = tmp_path / name
    f.write_bytes(gzip.open(os.path.join(HERE, "golden", name + ".gz"), "rb").read())
    return str(f)


def deterministic_randomize(x):
    """The logs pipeline's randomize_udf (benchmarks/logs/runtuplex.py) with a fixed replacement instead of random.choice."""
    return re.sub("^/~[^/]+", "/~" + "ab", x)


def test_reference_logs_strip_pipeline(gpu, monkeypatch, tmp_path):
    logs, ips = _golden(tmp_path, "logs.sample.txt"), _golden(tmp_path, "bad_ips_all.txt")

    def make(ctx):
        return (ctx.text(logs).map(ParseWithStrip).mapColumn("endpoint", deterministic_randomize)
                .join(ctx.csv(ips), "ip", "BadIPs"))
    split, whole, (splits, values) = run_both(monkeypatch, make, "tocsv", tmp_path)
    ctx = split[4]._ctx
    assert splits == 1 and ctx.metrics.text_rows > 0 and not any("falls back" in m for m in ctx._messages)
    assert values == sum(1 for _ in read_lines([logs], print))  # one column read per log line
    bad = set(read_lines([ips], print)[1:])
    want = [r for r in map(ParseWithStrip, read_lines([logs], print)) if r["ip"] in bad]
    assert len(split[0].decode().splitlines()) == len(want) + 1 == 3438


# ---- tplx_gpu_block_select against numpy ----------------------------------------------------------------------------------------
def _col(t, n, rng, option):
    if t == T_STR:
        vals = ["".join(rng.choice("abcxyzé") for _ in range(rng.randrange(0, 9))) for _ in range(n)]
    elif t == T_F64:
        vals = [rng.uniform(-1e9, 1e9) for _ in range(n)]
    elif t == T_BOOL:
        vals = [rng.random() < 0.5 for _ in range(n)]
    else:
        vals = [rng.randrange(-(1 << 63), 1 << 63) for _ in range(n)]
    if option:
        vals = [None if rng.random() < 0.3 else v for v in vals]
    col = backend.Column.from_values(vals, t)
    if option and col.valid is None:
        col.valid = backend.pack_valid(np.ones(n, bool))
    return col


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, (1 << 21) + 5])
@pytest.mark.parametrize("pattern", ["none", "all", "alternating", "random"])
def test_block_select_against_numpy(gpu, n, pattern):
    rng = random.Random(n * 7 + len(pattern))
    m = min(n, 4096)  # values for the big size repeat a 4096-row pattern, the selection does not
    types = [T_I64, T_F64, T_BOOL, T_STR]
    small = [_col(t, m, rng, opt) for opt in (False, True) for t in types]
    cols = []
    for c in small:
        reps = (n + m - 1) // m if m else 0
        if c.type == T_STR:
            vals = (c.to_values() * reps)[:n]
            cols.append(backend.Column.from_values(vals, T_STR))
            if c.valid is not None:
                cols[-1].valid = backend.pack_valid(np.tile(c.present(), reps)[:n]) if n else np.zeros(0, np.uint32)
        else:
            data = np.tile(c.data, reps)[:n] if n else c.data[:0]
            valid = None if c.valid is None else (backend.pack_valid(np.tile(c.present(), reps)[:n]) if n else np.zeros(0, np.uint32))
            cols.append(backend.Column(c.type, data, None, valid))
    keep = {"none": np.zeros(n, bool), "all": np.ones(n, bool), "alternating": np.arange(n) % 2 == 0,
            "random": np.random.default_rng(n).random(n) < 0.4}[pattern]
    words = backend.pack_valid(keep)
    if n & 31:
        words[-1] |= np.uint32(~((1 << (n & 31)) - 1) & 0xFFFFFFFF)  # bits past the last row are ignored
    blk = backend.Block.upload(0, cols, n)
    out = blk.select(words)
    blk.free()
    idx = np.flatnonzero(keep)
    assert out.n_rows == len(idx)
    for c, col in enumerate(cols):
        got = out.column(c, col.type)
        raw = out.validity(c)
        if col.valid is None:
            assert raw is None
        else:
            want_present = col.present()[idx]
            assert raw.tolist() == backend.pack_valid(want_present).tolist()  # tail bits zero
        if col.type == T_STR:
            o = col.offsets.astype(np.int64)
            lens = (o[1:] - o[:-1])[idx]
            want_off = np.zeros(len(idx) + 1, np.int64)
            np.cumsum(lens, out=want_off[1:])
            assert got.offsets.astype(np.int64).tolist() == want_off.tolist()
            want_bytes = b"".join(col.data[o[i]:o[i + 1]].tobytes() for i in idx[:50000]) if len(idx) <= 50000 else None
            if want_bytes is not None:
                assert got.data.tobytes() == want_bytes
            else:
                starts = o[:-1][idx]
                pos = np.repeat(starts - want_off[:-1], lens) + np.arange(int(want_off[-1]))
                assert np.array_equal(got.data, col.data[pos])
        else:
            assert np.array_equal(got.data.view(np.uint64), col.data[idx].view(np.uint64))
    out.free()
