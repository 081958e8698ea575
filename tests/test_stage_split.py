"""Stages split at the operators the device cannot compile (no device needed): the columns a CPython UDF reads from its row, where
a stage splits and which operators go with the CPython part, and the typing of the column such an operator makes.
GPU twin: tests/test_gpu_stage_split.py (the split stages run against plain Python)."""
import string

import pytest

import tuplex_b200 as tuplex
from tuplex_b200 import dataset
from tuplex_b200.context import typed_column
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR

NAMES = ["a", "b", "s", "f"]


def reads(udf, names=NAMES, resolvers=()):
    op = dataset.Op("withColumn", udf, column="new")
    op.resolvers = [(ValueError, r) for r in resolvers]
    return dataset._read_set(op, list(names), len(names))


def _helper(row):
    return row["a"]


def _def_udf(x):
    t = x["s"].split(" ")
    return t[0] + str(x[3])


def _def_rebinds(x):
    x = x["s"]
    return x


def test_read_set_constant_subscripts():
    assert reads(lambda x: x["s"].split(" ")[0]) == [2]
    assert reads(lambda x: x["a"] + x[1]) == [0, 1]
    assert reads(lambda x: round(x[-1], 2)) == [3]
    assert reads(lambda x: x[-4] * 2) == [0]
    assert reads(lambda x: 7) == []


def test_read_set_resolvers_add_their_columns():
    assert reads(lambda x: x["a"] // 0, resolvers=[lambda x: x["b"]]) == [0, 1]
    assert reads(lambda x: x["a"], resolvers=[lambda x: len(x)]) == [0, 1, 2, 3]


def test_read_set_def_udf():
    assert reads(_def_udf) == [2, 3]
    assert reads(_def_rebinds) == [0, 1, 2, 3]  # the parameter is rebound: every column


@pytest.mark.parametrize("udf", [
    lambda a, b, s, f: a + b,             # several parameters unpack the row
    lambda x: _helper(x),                 # the row passed to a helper
    lambda x: len(x),                     # the row itself
    lambda x: [v for v in x],             # iterated
    lambda x: x[x["a"]],                  # an index that is not a constant
    lambda x: x["nope"],                  # a name that is not a column
    lambda x: x[9],                       # an index outside the row
    lambda x: (lambda x: x)(x["a"]),      # shadowed by an inner parameter
], ids=["multi_param", "helper", "len", "iterate", "dynamic_index", "unknown_name", "out_of_range", "shadowed"])
def test_read_set_any_other_use_reads_every_column(udf):
    assert reads(udf) == [0, 1, 2, 3]


def test_read_set_of_a_one_column_row():
    assert reads(lambda v: v + 1, names=["v"]) == [0]  # the parameter is the value itself


def test_read_set_from_source_strings():
    assert reads("lambda x: x['b'] * 2") == [1]
    assert reads("def f(x):\n    return x['s'] + x['s']\n") == [2]


# ---- planning ------------------------------------------------------------------------------------------------------------------
def _ops(ds):
    return list(ds._ops)


def test_split_at_first_unsupported_operator():
    ctx = tuplex.Context()
    ds = (ctx.parallelize([(1, 2, "a b", 1.5)], columns=NAMES)
          .withColumn("g", lambda x: x["a"] + x["b"])
          .mapColumn("s", lambda v: string.capwords(v))
          .filter(lambda x: x["g"] > 0)
          .mapColumn("f", lambda v: round(v, 2)))
    ops = _ops(ds)
    assert dataset._split_point(ctx, ds._source, ops) == 1
    # the remainder is planned the same way again over the schema after U: its second unsupported operator splits it once more
    rest = ops[2:]
    sc_src = ctx._source_from_rows([(1, 2, "A B", 1.5, 3)], NAMES + ["g"])
    assert dataset._split_point(ctx, sc_src, rest) == 1


def test_resolvers_and_ignores_go_with_the_interpreter_operator():
    ctx = tuplex.Context()
    ds = (ctx.parallelize([(1, 2, "a b", 1.5)], columns=NAMES)
          .filter(lambda x: x["a"] > 0)
          .withColumn("w", lambda x: x["s"].split(" ")[1]).resolve(IndexError, lambda x: "?").ignore(KeyError)
          .withColumn("n", lambda x: len(x["w"])))
    ops = _ops(ds)
    k = dataset._split_point(ctx, ds._source, ops)
    assert k == 1
    assert [c for c, _ in ops[k].resolvers] == [IndexError] and ops[k].ignores == [KeyError]


def test_no_split_without_a_device_row_operator():
    ctx = tuplex.Context()
    only_u = ctx.parallelize([(1, 2, "a b", 1.5)], columns=NAMES).mapColumn("s", lambda v: string.capwords(v))
    assert dataset._split_point(ctx, only_u._source, _ops(only_u)) is None
    # selectColumns / renameColumn and the endpoint are not row operators of their own
    ds = only_u.selectColumns(["a", "s"]).renameColumn("a", "z")
    assert dataset._split_point(ctx, ds._source, _ops(ds)) is None


def test_no_split_where_results_cannot_stay_on_the_device():
    rows = [(1, 2, "a b", 1.5), (3, 4, "c d", 2.5)]
    pipe = lambda ds: ds.withColumn("g", lambda x: x["a"] + 1).mapColumn("s", lambda v: string.capwords(v))  # noqa: E731
    for conf in ({"tuplex.gpu.optionColumns": False}, {"tuplex.gpu.devices": "0,0"}):
        ctx = tuplex.Context(conf)
        ds = pipe(ctx.parallelize(rows, columns=NAMES))
        assert dataset._split_point(ctx, ds._source, _ops(ds)) is None
    ctx = tuplex.Context()
    ds = pipe(ctx.parallelize(rows + [("x", 2, "e f", 1.0)], columns=NAMES))  # a fallback row
    assert ds._source.fallback and dataset._split_point(ctx, ds._source, _ops(ds)) is None


def test_no_split_when_the_stage_compiler_cannot_be_built(monkeypatch):
    class NoCompiler:
        def __init__(self, *a, **k):
            raise dataset.UnsupportedUDF("no compiler")
    monkeypatch.setattr(dataset, "StageCompiler", NoCompiler)
    ctx = tuplex.Context()
    ds = ctx.parallelize([(1, 2, "a b", 1.5)], columns=NAMES).withColumn("g", lambda x: x["a"] + 1).mapColumn("s", string.capwords)
    assert dataset._split_point(ctx, ds._source, _ops(ds)) is None


def test_compiled_stage_has_no_split_point():
    ctx = tuplex.Context()
    ds = ctx.parallelize([(1, 2, "a b", 1.5)], columns=NAMES).withColumn("g", lambda x: x["a"] + 1)
    assert dataset._split_point(ctx, ds._source, _ops(ds)) is None


# ---- the new column's type -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("values,t,nullable", [
    ([1, 2, -3], T_I64, False),
    ([1.5, 2.0], T_F64, False),
    (["x", ""], T_STR, False),
    ([True, False], T_BOOL, False),
    (["x", None, "y"], T_STR, True),
    ([None, 4], T_I64, True),
    ([-(1 << 63), (1 << 63) - 1], T_I64, False),
])
def test_typed_column(values, t, nullable):
    col = typed_column(values)
    assert col.type == t and (col.valid is not None) == nullable
    assert col.to_values() == values


@pytest.mark.parametrize("values", [[1, 2.5], [1, True], ["x", 1], [None, None], [], [1 << 63], [1, -(1 << 63) - 1], [(1, 2)]],
                         ids=["int_float", "int_bool", "str_int", "all_none", "empty", "beyond_i64", "below_i64", "tuple"])
def test_typed_column_gives_up(values):
    assert typed_column(values) is None


def test_typed_column_is_the_source_typing():
    """The rule is the one _source_from_rows applies to a column: the same values make the same column there."""
    ctx = tuplex.Context()
    for values in ([1, None, 3], ["a", None], [2.5, 1.0, None]):
        src = ctx._source_from_rows([(v, 0) for v in values], ["c", "d"])
        col = typed_column(values)
        assert not src.fallback and src.cols[0].type == col.type and src.cols[0].to_values() == col.to_values()
    src = ctx._source_from_rows([(1, 0), (2.5, 0), (3, 0)], ["c", "d"])
    assert src.fallback and typed_column([1, 2.5, 3]) is None  # a row the source leaves outside the normal case: give up
