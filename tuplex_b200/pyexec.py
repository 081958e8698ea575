"""CPython row pipeline: the slow path.

The reference re-runs exception rows through a generated pure-Python pipeline under the GIL and merges
the results back by row number (tuplex/core/src/physical/ResolveTask.cc:389,702-1258;
tuplex/core/include/physical/PythonPipelineBuilder.h:23-110). The GPU backend hands its exception
records to exactly this path; nothing here runs for rows that stay on the normal case.
This is also what executes a whole operator chain when a UDF is outside the GPU op set
(`resolveWithInterpreterOnly`-style).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

from .ir import C

# exception class -> reference code (tuplex/utils/include/ExceptionCodes.h:24-120)
EXC_CODES = {
    "IndexError": 111, "KeyError": 112, "TypeError": 129, "ValueError": 135, "ZeroDivisionError": 136,
    "AttributeError": 106, "AssertionError": 105, "OverflowError": 118, "ArithmeticError": 102, "LookupError": 104,
    "Exception": 101, "BaseException": 100, "RuntimeError": 121, "NameError": 115, "UnboundLocalError": 130,
    "UnicodeError": 131, "NotImplementedError": 116,
}
CODE_NAMES = {v: k for k, v in EXC_CODES.items()}
CODE_NAMES.update({7: "NormalCaseViolation", 50: "NullError", 80: "PythonParallelize", 70: "BadParseStringInput"})


def exception_code(e: BaseException) -> int:
    for cls in type(e).__mro__:
        if cls.__name__ in EXC_CODES:
            return EXC_CODES[cls.__name__]
    return 101


class Row(tuple):
    """A row as a UDF sees it: indexable by position and by column name (python/tuplex/dataset.py semantics)."""
    names: Optional[Tuple[Optional[str], ...]] = None

    def __new__(cls, values, names=None):
        r = super().__new__(cls, values)
        r.names = tuple(names) if names is not None else None
        return r

    def __getitem__(self, k):
        if isinstance(k, str):
            if not self.names or k not in self.names:
                raise KeyError(k)
            return tuple.__getitem__(self, self.names.index(k))
        return tuple.__getitem__(self, k)

    def keys(self):
        return list(self.names or ())


class Op:
    """Logical operator (tuplex/core/include/logical/*Operator.h); ids start at 100000 like
    LogicalOperator::logicalOperatorIDGenerator (tuplex/core/include/logical/LogicalOperator.h:52-59)."""
    _next_id = 100000

    def __init__(self, kind: str, udf=None, column=None, columns=None, extra=None):
        self.kind = kind
        self.udf = udf
        self.column = column
        self.columns = columns
        self.extra = extra
        self.id = Op._next_id
        Op._next_id += 1
        self.resolvers: List[Tuple[type, Any]] = []   # (exception class, resolver udf) attached by .resolve()
        self.ignores: List[type] = []                 # attached by .ignore()


class Dropped(Exception):
    pass


_SRC_CACHE: dict = {}


def udf_from_source(src: str):
    """A UDF given as source text (the reference's UDF("lambda x: ...") / UDF("def f(x): ...")): compiled once."""
    fn = _SRC_CACHE.get(src)
    if fn is None:
        text = src.strip()
        if text.startswith("def "):
            import textwrap
            ns: dict = {}
            exec(textwrap.dedent(src).strip().expandtabs(4), ns)  # noqa: S102 — user code, like any UDF
            fns = [v for k, v in ns.items() if callable(v) and not k.startswith("__")]
            fn = fns[-1]
        else:
            fn = eval(text)  # noqa: S307
        _SRC_CACHE[src] = fn
    return fn


def _call(udf, value, names):
    """Call a UDF with Tuplex's argument convention: one column -> the value itself, many -> a Row;
    a multi-parameter lambda unpacks the row."""
    if isinstance(udf, str):
        udf = udf_from_source(udf)
    if isinstance(value, tuple):
        n = udf.__code__.co_argcount
        if n > 1 and n == len(value):
            return udf(*value)
        return udf(Row(value, names))
    return udf(value)


def _apply_with_resolvers(op: Op, fn):
    try:
        return fn(op.udf)
    except Exception as e:  # noqa: BLE001
        for cls in op.ignores:
            if isinstance(e, cls):
                raise Dropped() from None
        for cls, res in op.resolvers:
            if isinstance(e, cls):
                return fn(res)
        raise


def call_op(op: Op, value, names: List[Optional[str]]):
    """What one row gives the UDF of a map / filter / withColumn / mapColumn operator, with its resolvers and ignores applied: the
    map's result, the filter's verdict, the new column's value. Raises Dropped (an ignored class) or the UDF's exception."""
    if op.kind == "mapColumn":
        vals = list(value) if isinstance(value, tuple) else [value]
        i = names.index(op.column) if isinstance(op.column, str) else op.column
        return _apply_with_resolvers(op, lambda f: (udf_from_source(f) if isinstance(f, str) else f)(vals[i]))
    return _apply_with_resolvers(op, lambda f: _call(f, value, names))


def run_row(ops: Sequence[Op], value, names: List[Optional[str]]):
    """Run one row through the operator chain in CPython.
    Returns (value, names) or raises: Dropped (filtered / ignored) or the UDF's exception (annotated with .tplx_op)."""
    names = list(names)
    for op in ops:
        try:
            if op.kind == "map":
                res = call_op(op, value, names)
                if isinstance(res, dict):
                    names = list(res.keys())
                    res = tuple(res.values())
                    value = res if len(res) != 1 else res[0]
                elif isinstance(res, tuple):
                    names = [None] * len(res)
                    value = tuple(res) if len(res) != 1 else res[0]
                else:
                    names = [None]
                    value = res
            elif op.kind == "filter":
                keep = call_op(op, value, names)
                if not keep:
                    raise Dropped()
            elif op.kind == "withColumn":
                res = call_op(op, value, names)
                vals = list(value) if isinstance(value, tuple) else [value]
                if op.column in names:
                    vals[names.index(op.column)] = res
                else:
                    vals.append(res)
                    names.append(op.column)
                value = tuple(vals) if len(vals) != 1 else vals[0]
            elif op.kind == "mapColumn":
                vals = list(value) if isinstance(value, tuple) else [value]
                vals[names.index(op.column) if isinstance(op.column, str) else op.column] = call_op(op, value, names)
                value = tuple(vals) if len(vals) != 1 else vals[0]
            elif op.kind == "selectColumns":
                vals = list(value) if isinstance(value, tuple) else [value]
                idx = [names.index(c) if isinstance(c, str) else (c % len(vals)) for c in op.columns]
                vals = [vals[i] for i in idx]
                names = [names[i] for i in idx]
                value = tuple(vals) if len(vals) != 1 else vals[0]
            elif op.kind == "renameColumn":
                i = names.index(op.column) if isinstance(op.column, str) else op.column
                names[i] = op.extra
            else:
                raise NotImplementedError(op.kind)
        except Dropped:
            raise
        except Exception as e:  # noqa: BLE001
            if not hasattr(e, "tplx_op"):
                e.tplx_op = op.id
            raise
    return value, names
