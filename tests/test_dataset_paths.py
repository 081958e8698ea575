"""DataSet pipelines through both execution paths, against plain-Python references written out in this file.

Every pipeline mixes normal-case rows, rows whose UDF raises (some resolved, some ignored, some left as exceptions) and fallback
rows that do not fit the normal-case schema. On the device path the stage runs on the GPU and only the rows that leave the normal
case run in CPython; on the CPython path (a UDF outside the GPU op set, or no stage compiler) the whole stage does. Both must give
the reference's rows and exception counts. The CPU part runs the CPython path only."""
from collections import Counter

import pytest

import tuplex_b200 as tuplex
from tuplex_b200 import backend, dataset, frontend

N = 5000
BLOCK_ROWS = 1000  # five blocks per stage on the device path


def make_rows(n=N, fallback=True):
    """(a, b, s) rows; b == 0 in every 7th row. Fallback rows: a float in a, a str in b, an int in s."""
    rows = []
    for i in range(n):
        if fallback and i % 101 == 50:
            rows.append((i + 0.5, i % 7 - 3, "f%d" % (i % 3)))
        elif fallback and i % 101 == 70:
            rows.append((i, str(i % 7), "g"))
        elif fallback and i % 101 == 90:
            rows.append((i, i % 7 - 3, i % 4))
        else:
            rows.append((i, i % 7 - 3, "k%d" % (i % 5)))
    return rows


def exception_counts(ds):
    """ds.exception_counts keyed by (position of the operator in the pipeline, exception name): every run builds its own
    operators, with new ids."""
    pos = {op.id: i for i, op in enumerate(ds._ops)}
    return {(pos[op_id], name): n for (op_id, name), n in ds.exception_counts.items()}


def case_rows(ctx, data):
    """map + resolve, filter, withColumn, mapColumn, selectColumns, renameColumn -> collect."""
    ds = (ctx.parallelize(data, columns=["a", "b", "s"])
          .map(lambda x: {"a": x["a"], "q": x["a"] // x["b"], "s": x["s"]})
          .resolve(ZeroDivisionError, lambda x: {"a": x["a"], "q": -1, "s": x["s"]})
          .filter(lambda x: x["q"] % 3 != 1)
          .withColumn("t", lambda x: x["q"] * 2 + len(x["s"]))
          .mapColumn("s", lambda v: v.upper())
          .selectColumns(["t", "s", "a"])
          .renameColumn("s", "S"))
    rows, counts = [], Counter()
    for a, b, s in data:
        try:
            q = a // b
        except ZeroDivisionError:
            q = -1
        except TypeError:
            counts[(0, "TypeError")] += 1
            continue
        if q % 3 == 1:
            continue
        try:
            t = q * 2 + len(s)
        except TypeError:
            counts[(2, "TypeError")] += 1
            continue
        rows.append((t, s.upper(), a))
    return ds, rows, counts


def case_ignore(ctx, data):
    """withColumn + ignore, a withColumn whose exceptions stay, mapColumn, selectColumns -> collect."""
    ds = (ctx.parallelize(data, columns=["a", "b", "s"])
          .withColumn("q", lambda x: x["a"] // x["b"]).ignore(ZeroDivisionError)
          .withColumn("r", lambda x: 100 // (x["a"] % 13))
          .mapColumn("b", lambda v: v * 10)
          .selectColumns(["q", "r", "b", "s"]))
    rows, counts = [], Counter()
    for a, b, s in data:
        try:
            q = a // b
        except ZeroDivisionError:
            continue
        except TypeError:
            counts[(0, "TypeError")] += 1
            continue
        try:
            r = 100 // (a % 13)
        except ZeroDivisionError:
            counts[(1, "ZeroDivisionError")] += 1
            continue
        rows.append((q, r, b * 10, s))
    return ds, rows, counts


def case_aggregate(ctx, data):
    """map + resolve -> aggregate whose UDF reads columns by name and raises for int s."""
    ds = (ctx.parallelize(data, columns=["a", "b", "s"])
          .map(lambda x: {"q": x["a"] // x["b"], "s": x["s"]})
          .resolve(ZeroDivisionError, lambda x: {"q": 7, "s": x["s"]})
          .aggregate(lambda p, r: p + r, lambda acc, x: acc + x["q"] * len(x["s"]), 0))
    total, counts = 0, Counter()
    for a, b, s in data:
        try:
            q = a // b
        except ZeroDivisionError:
            q = 7
        except TypeError:
            counts[(0, "TypeError")] += 1
            continue
        try:
            total += q * len(s)
        except TypeError:
            counts[(1, "TypeError")] += 1
    return ds, [total], counts


def case_aggregate_by_key(ctx, data):
    """map + ignore -> aggregateByKey whose UDF raises for int s."""
    ds = (ctx.parallelize(data, columns=["a", "b", "s"])
          .map(lambda x: {"k": x["a"] % 4, "q": x["a"] // x["b"], "s": x["s"]}).ignore(ZeroDivisionError)
          .aggregateByKey(lambda p, r: p + r, lambda acc, x: acc + (x["q"] + len(x["s"])), 0, ["k"]))
    groups, counts = {}, Counter()
    for a, b, s in data:
        try:
            q = a // b
        except ZeroDivisionError:
            continue
        except TypeError:
            counts[(0, "TypeError")] += 1
            continue
        try:
            groups[a % 4] = groups.get(a % 4, 0) + q + len(s)
        except TypeError:
            counts[(1, "TypeError")] += 1
    return ds, sorted(groups.items()), counts


def case_unique(ctx, data):
    """map + resolve -> unique."""
    ds = (ctx.parallelize(data, columns=["a", "b", "s"])
          .map(lambda x: (x["a"] // x["b"] % 4, x["s"]))
          .resolve(ZeroDivisionError, lambda x: (-1, x["s"]))
          .unique())
    seen, counts = set(), Counter()
    for a, b, s in data:
        try:
            seen.add((a // b % 4, s))
        except ZeroDivisionError:
            seen.add((-1, s))
        except TypeError:
            counts[(0, "TypeError")] += 1
    return ds, sorted(seen, key=repr), counts


CASES = [case_rows, case_ignore, case_aggregate, case_aggregate_by_key, case_unique]


class _NoCompiler:
    def __init__(self, *args, **kwargs):
        raise frontend.UnsupportedUDF("every stage on the CPython path")


def _collect(ds, case):
    rows = ds.collect()
    return sorted(rows, key=repr) if case is case_unique else rows


# ---- CPU: the CPython path ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.__name__)
def test_cpython_path_equals_reference(case, monkeypatch):
    monkeypatch.setattr(dataset, "StageCompiler", _NoCompiler)
    ctx = tuplex.Context()
    ds, want_rows, want_counts = case(ctx, make_rows())
    assert ds._source.fallback  # the source has rows outside the normal case
    assert _collect(ds, case) == want_rows
    assert exception_counts(ds) == dict(want_counts)
    assert any("falls back" in m for m in ctx._messages)


def _sorted_stage(ctx):
    """A stage with a UDF outside the GPU op set (sorted): it runs on the CPython path."""
    return ctx.parallelize([(1, 2), (3, 4), (5, 6)], columns=["a", "b"]).map(
        lambda x: {"a": x["a"], "m": sorted([x["a"], x["b"]])[0]})


def test_cpython_path_aggregate_udf_gets_a_row():
    ds = _sorted_stage(tuplex.Context()).aggregate(lambda a, b: a + b, lambda a, x: a + x["a"], 0)
    assert ds.collect() == [9]
    assert exception_counts(ds) == {}


def test_cpython_path_aggregate_by_key_counts_udf_exceptions():
    ds = _sorted_stage(tuplex.Context()).aggregateByKey(lambda a, b: a + b, lambda a, x: a + 10 // (x["a"] - 3), 0, ["a"])
    assert ds.collect() == [(1, -5), (5, 5)]
    assert exception_counts(ds) == {(1, "ZeroDivisionError"): 1}  # counted under the aggregateByKey operator


# ---- GPU: the device path and the CPython path ------------------------------------------------------------------------------
def _device_ctx():
    return tuplex.Context({"tuplex.gpu.blockRows": BLOCK_ROWS})


def _on_both_paths(monkeypatch, run):
    """run(ctx) once on the device path and once with every stage on the CPython path."""
    dctx = _device_ctx()
    on_device = run(dctx)
    assert not [m for m in dctx._messages if "falls back" in m], dctx._messages
    with monkeypatch.context() as mp:
        mp.setattr(dataset, "StageCompiler", _NoCompiler)
        on_cpython = run(_device_ctx())
    return on_device, on_cpython


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.__name__)
def test_device_path_equals_cpython_path_and_reference(gpu, case, monkeypatch):
    data = make_rows()
    _, want_rows, want_counts = case(_device_ctx(), data)

    def run(ctx):
        ds = case(ctx, data)[0]
        return _collect(ds, case), exception_counts(ds)
    on_device, on_cpython = _on_both_paths(monkeypatch, run)
    assert on_device == on_cpython == (want_rows, dict(want_counts))


def _csv_text(names, rows):
    def cell(v):
        return "%.8f" % v if isinstance(v, float) else str(v)
    return "".join(",".join(cell(v) for v in r) + "\n" for r in [tuple(names)] + rows)


@pytest.mark.gpu
@pytest.mark.parametrize("fallback", [False, True], ids=["device_merge", "host_formatter"])
def test_tocsv_on_both_paths(gpu, tmp_path, monkeypatch, fallback):
    """Without fallback rows the device merges the resolved exception rows back in (K9, one merge per block) and writes the
    text; with fallback rows the host formats the merged rows."""
    calls = []
    orig = backend.Result.merge_resolved
    monkeypatch.setattr(backend.Result, "merge_resolved", lambda self, *a, **k: (calls.append(1), orig(self, *a, **k))[1])
    data = make_rows(fallback=fallback)
    _, want_rows, want_counts = case_rows(_device_ctx(), data)
    paths = iter(["device.csv", "cpython.csv"])

    def run(ctx):
        ds = case_rows(ctx, data)[0]
        out = tmp_path / next(paths)
        ds.tocsv(str(out))
        return out.read_text(), exception_counts(ds)
    on_device, on_cpython = _on_both_paths(monkeypatch, run)
    assert len(calls) == (0 if fallback else N // BLOCK_ROWS)
    assert on_device == on_cpython == (_csv_text(["t", "S", "a"], want_rows), dict(want_counts))
