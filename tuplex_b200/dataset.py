"""DataSet — mirror of the reference's python API for the hot path
(tuplex/python/tuplex/dataset.py: map/filter/collect :49-123, withColumn/mapColumn/selectColumns :201-290,
aggregate/aggregateByKey :593-705) executed by the GPU backend.

Planning is the small plan->stage-descriptor lowering SURVEY.md §2 row 3 calls for: consecutive
map/filter/withColumn/mapColumn/selectColumns/renameColumn operators fuse into one stage (the reference
fuses the same operators into one TransformStage, tuplex/core/src/physical/PhysicalPlan.cc:60-420); an
aggregate ends a stage. Execution = LocalBackend::executeTransformStage's job
(tuplex/core/src/ee/local/LocalBackend.cc:815-1252): run the normal case, collect exception rows, resolve
them on the CPython path, merge in order.
"""
from __future__ import annotations

import struct
from collections import Counter
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import backend, ir, pyexec
from .backend import Column
from .frontend import StageCompiler, UnsupportedUDF
from .ir import C, T_BOOL, T_F64, T_I64, T_STR
from .pyexec import Dropped, Op


def _clone_op(op: Op) -> Op:
    """Same operator (same id: exception counts are keyed by it) with its own resolver / ignore lists. The reference adds a
    separate ResolveOperator / IgnoreOperator node and leaves the parent plan untouched (python/tuplex/dataset.py:344-389)."""
    import copy
    c = copy.copy(op)
    c.resolvers = list(op.resolvers)
    c.ignores = list(op.ignores)
    return c


class Source:
    """Input of a plan: normal-case column block + rows that did not fit the normal-case schema
    (PythonContext::parallelize fallback rows, tuplex/python/src/PythonContext.cc:178-204)."""

    def __init__(self, cols: List[Column], names: List[Optional[str]], n_rows: int, orig_index: Optional[np.ndarray],
                 fallback: List[Tuple[int, Any]], total_rows: int):
        self.cols = cols
        self.names = names
        self.n_rows = n_rows
        self.orig_index = orig_index  # original list position of each normal row (None = identity)
        self.fallback = fallback      # (original position, python object)
        self.total_rows = total_rows


class JoinSpec:
    """A JoinOperator of the logical plan (tuplex/core/src/logical/JoinOperator.cc): two upstream datasets, the key column on each
    side, inner or left, and the prefixes / suffixes applied to the column names of each side."""

    def __init__(self, left: "DataSet", right: "DataSet", left_col: str, right_col: str, kind: str, left_prefix: str, left_suffix: str,
                 right_prefix: str, right_suffix: str):
        self.left, self.right = left, right
        self.left_col, self.right_col = left_col, right_col
        self.kind = kind  # "inner" | "left"
        self.left_prefix, self.left_suffix = left_prefix, left_suffix
        self.right_prefix, self.right_suffix = right_prefix, right_suffix

    def key_indices(self, lnames, rnames):
        if self.left_col not in lnames:
            raise ValueError(f"column '{self.left_col}' not found in left dataset for join.")  # JoinOperator.cc:99-102
        if self.right_col not in rnames:
            raise ValueError(f"column '{self.right_col}' not found in right dataset for join.")
        return lnames.index(self.left_col), rnames.index(self.right_col)

    def names(self, lnames, rnames):
        """| left columns except the key | key (left name) | right columns except the key |  (JoinOperator.cc:163-184)"""
        li, ri = self.key_indices(lnames, rnames)
        deco = lambda n, p, s: None if n is None else p + n + s  # noqa: E731
        return ([deco(n, self.left_prefix, self.left_suffix) for i, n in enumerate(lnames) if i != li] +
                [deco(lnames[li], self.left_prefix, self.left_suffix)] +
                [deco(n, self.right_prefix, self.right_suffix) for i, n in enumerate(rnames) if i != ri])

    def build_right(self) -> bool:
        """JoinOperator::buildRight (core/include/logical/JoinOperator.h:62-69): a left join always builds on the right side,
        an inner join on the side with the smaller cost."""
        return self.kind == "left" or self.left._cost() >= self.right._cost()


class DataSet:
    def __init__(self, ctx, source: Optional[Source], ops: Sequence[Op] = (), parent: Optional["DataSet"] = None,
                 join: Optional[JoinSpec] = None):
        self._ctx = ctx
        self._source = source
        self._ops: List[Op] = list(ops)
        self._parent = parent  # upstream DataSet whose result is this one's source (after an aggregate)
        self._join = join      # this dataset's source is the join of two upstream datasets
        self._last_exceptions: Counter = Counter()

    # ---- lazy operators ---------------------------------------------------------------------------
    def _with(self, op: Op) -> "DataSet":
        return DataSet(self._ctx, self._source, self._ops + [op], self._parent, self._join)

    def join(self, dsRight: "DataSet", leftKeyColumn: str, rightKeyColumn: str, prefixes=None, suffixes=None) -> "DataSet":
        """(inner) join with another dataset on one key column per side (python/tuplex/dataset.py:384-440)."""
        return self._make_join(dsRight, leftKeyColumn, rightKeyColumn, prefixes, suffixes, "inner")

    def leftJoin(self, dsRight: "DataSet", leftKeyColumn: str, rightKeyColumn: str, prefixes=None, suffixes=None) -> "DataSet":
        """left (outer) join: rows of this dataset without a partner keep None in the right columns (python/tuplex/dataset.py:442-498)."""
        return self._make_join(dsRight, leftKeyColumn, rightKeyColumn, prefixes, suffixes, "left")

    def _make_join(self, dsRight, leftKeyColumn, rightKeyColumn, prefixes, suffixes, kind):
        if not isinstance(dsRight, DataSet):
            raise TypeError("dsRight must be a DataSet")
        lp = ls = rp = rs = ""
        if prefixes:
            prefixes = tuple(prefixes)
            assert len(prefixes) == 2, "prefixes must be a sequence of 2 elements!"
            lp, rp = prefixes[0] or "", prefixes[1] or ""
        if suffixes:
            suffixes = tuple(suffixes)
            assert len(suffixes) == 2, "suffixes must be a sequence of 2 elements!"
            ls, rs = suffixes[0] or "", suffixes[1] or ""
        spec = JoinSpec(self, dsRight, leftKeyColumn, rightKeyColumn, kind, lp, ls, rp, rs)
        spec.names(self._plan_names()[1], dsRight._plan_names()[1])  # unknown key columns are reported when the join is declared
        return DataSet(self._ctx, None, [], None, spec)

    def _cost(self) -> int:
        """LogicalOperator::cost (core/include/logical/LogicalOperator.h:197-204): sources report their row count
        (ParallelizeOperator.cc:121-129, FileInputOperator.cc:533-536), every other operator the sum over its parents."""
        if self._join is not None:
            return self._join.left._cost() + self._join.right._cost()
        if self._parent is not None:
            return self._parent._cost()
        src = self._source
        if src is None:
            return 0
        if hasattr(src, "chunks"):  # CSV source: data rows = line ends of the files (the reference estimates from a sample)
            return int(sum(int(np.count_nonzero(a == 10)) for a in getattr(src, "files", [])))
        return int(src.total_rows)

    def map(self, ftor):
        return self._with(Op("map", ftor))

    def filter(self, ftor):
        return self._with(Op("filter", ftor))

    def withColumn(self, column, ftor):
        return self._with(Op("withColumn", ftor, column=column))

    def mapColumn(self, column, ftor):
        return self._with(Op("mapColumn", ftor, column=column))

    def selectColumns(self, columns):
        if not isinstance(columns, (list, tuple)):
            columns = [columns]
        return self._with(Op("selectColumns", columns=list(columns)))

    def renameColumn(self, key, newColumnName):
        return self._with(Op("renameColumn", column=key, extra=newColumnName))

    def resolve(self, eclass, ftor):
        if not self._ops:
            raise ValueError("resolve() needs a preceding operator")
        ds = DataSet(self._ctx, self._source, self._ops, self._parent, self._join)
        ds._ops[-1] = _clone_op(ds._ops[-1])  # the parent DataSet (and its other branches) keep the operator without this resolver
        ds._ops[-1].resolvers.append((eclass, ftor))
        return ds

    def ignore(self, eclass):
        if not self._ops:
            raise ValueError("ignore() needs a preceding operator")
        ds = DataSet(self._ctx, self._source, self._ops, self._parent, self._join)
        ds._ops[-1] = _clone_op(ds._ops[-1])
        ds._ops[-1].ignores.append(eclass)
        return ds

    def aggregate(self, combine, aggregate, initial_value):
        return self._with(Op("aggregate", udf=aggregate, extra=(combine, initial_value)))

    def aggregateByKey(self, combine, aggregate, initial_value, key_columns):
        if not isinstance(key_columns, (list, tuple)):
            key_columns = [key_columns]
        return self._with(Op("aggregateByKey", udf=aggregate, columns=list(key_columns), extra=(combine, initial_value)))

    def unique(self):
        return self._with(Op("unique"))

    def cache(self, store_specialized=True):
        rows, names = self._execute()
        return self._ctx._dataset_from_rows(rows, names)

    # ---- actions ------------------------------------------------------------------------------------
    def collect(self):
        rows, _ = self._execute()
        return rows

    def take(self, nrows=5):
        rows, _ = self._execute()
        return rows[:nrows] if nrows >= 0 else rows

    def show(self, nrows=None):
        rows, names = self._execute()
        if any(names):
            print(" | ".join(str(n) for n in names))
        for r in rows[: (nrows if nrows is not None else len(rows))]:
            print(r)

    def tocsv(self, path, part_size=0, num_rows=None, num_parts=0, part_name_generator=None, null_value=None, header=True):
        """CSV sink (python/tuplex/dataset.py:502-560). Rows are formatted like the reference's row writer
        (fast_csvwriter, PipelineBuilder.cc:1550-1722): on the device (K7, tplx_gpu_result_csv) when the last stage ran
        there without rows from the interpreter path, else by the host twin `_csv_cell`."""
        import os
        self._csv_sink = []
        try:
            rows, names = self._execute(sink="csv")
            chunks = self._csv_sink
        finally:
            self._csv_sink = None
        os.makedirs(path, exist_ok=True) if not path.endswith(".csv") else None
        fn = path if path.endswith(".csv") else os.path.join(path, "part0.csv")
        with open(fn, "wb") as fp:
            if header and any(names):
                fp.write((",".join(_csv_cell(str(n)) for n in names) + "\n").encode())
            if rows is None:
                for ch in chunks:
                    fp.write(ch)
            else:
                for r in rows:
                    vals = r if isinstance(r, tuple) else (r,)
                    fp.write((",".join(_csv_cell(v, null_value) for v in vals) + "\n").encode())

    @property
    def columns(self):
        _, names = self._plan_names()
        return names

    @property
    def types(self):
        """Output schema as a list of `typing` types (python/tuplex/dataset.py:374-382), from the plan alone where the operators
        compile for the device (Option[T] columns -> typing.Optional[T]); datasets behind a join / an interpreter-path stage are
        typed from their first rows."""
        import typing
        py = {T_I64: int, T_F64: float, T_BOOL: bool, T_STR: str}
        if self._join is None and self._parent is None and self._source is not None and not hasattr(self._source, "chunks"):
            try:
                sc = StageCompiler([c.type for c in self._source.cols], self._source.names, _option_cols(self._source.cols))
                for o in self._ops:
                    if o.kind == "map":
                        sc.add_map(o.udf, o.id)
                    elif o.kind == "filter":
                        sc.add_filter(o.udf, o.id)
                    elif o.kind == "withColumn":
                        sc.add_with_column(o.column, o.udf, o.id)
                    elif o.kind == "mapColumn":
                        sc.add_map_column(o.column, o.udf, o.id)
                    elif o.kind == "selectColumns":
                        sc.add_select(o.columns, o.id)
                    elif o.kind == "renameColumn":
                        sc.add_rename(o.column, o.extra, o.id)
                    else:
                        raise UnsupportedUDF("endpoint")
                return [typing.Optional[py[v.type]] if v.null is not None else py[v.type] for v in sc.row]
            except (UnsupportedUDF, KeyError):
                pass
        rows = self.take(64)
        if not rows:
            return None
        tup = [r if isinstance(r, tuple) else (r,) for r in rows]
        out = []
        for c in range(len(tup[0])):
            ts = {type(r[c]) for r in tup if len(r) > c and r[c] is not None}
            t = ts.pop() if len(ts) == 1 else typing.Any
            out.append(typing.Optional[t] if any(len(r) > c and r[c] is None for r in tup) else t)
        return out

    @property
    def exception_counts(self):
        return dict(self._last_exceptions)

    # ---- planning + execution -------------------------------------------------------------------------
    def _plan_names(self):
        """Column names from the logical plan alone (the reference derives them without executing,
        python/tuplex/dataset.py:720-735): operators are replayed over names only."""
        if self._join is not None:
            names = self._join.names(self._join.left._plan_names()[1], self._join.right._plan_names()[1])
        elif self._parent is not None:
            _, names = self._parent._plan_names()
            names = list(names)
        else:
            names = list(self._source.names) if self._source is not None else []
        for op in self._ops:
            if op.kind == "withColumn":
                if op.column not in names:
                    names = names + [op.column]
            elif op.kind == "selectColumns":
                names = [c if isinstance(c, str) else names[c] for c in op.columns]
            elif op.kind == "renameColumn":
                names = [op.extra if (n == op.column or (isinstance(op.column, int) and i == op.column % max(len(names), 1))) else n
                         for i, n in enumerate(names)]
            elif op.kind == "map":
                names = self._names_after_map(op, names)
            elif op.kind == "aggregate":
                init = op.extra[1]
                names = [None] * (len(init) if isinstance(init, (tuple, list)) else 1)
            elif op.kind == "aggregateByKey":
                init = op.extra[1]
                names = [c if isinstance(c, str) else names[c] for c in op.columns] + [None] * (len(init) if isinstance(init, (tuple, list)) else 1)
        return None, names

    def _names_after_map(self, op, names):
        """Compile (never run) the operator chain up to `op` to learn the shape its map() returns; UDFs outside the GPU op set
        fall back to reading the UDF's return expression."""
        if self._parent is None and self._source is not None and len(self._source.cols) == len(names):
            try:
                sc = StageCompiler([c.type for c in self._source.cols], self._source.names, _option_cols(self._source.cols))
                for o in self._ops:
                    if o.kind == "map":
                        sc.add_map(o.udf, o.id)
                    elif o.kind == "filter":
                        sc.add_filter(o.udf, o.id)
                    elif o.kind == "withColumn":
                        sc.add_with_column(o.column, o.udf, o.id)
                    elif o.kind == "mapColumn":
                        sc.add_map_column(o.column, o.udf, o.id)
                    elif o.kind == "selectColumns":
                        sc.add_select(o.columns, o.id)
                    elif o.kind == "renameColumn":
                        sc.add_rename(o.column, o.extra, o.id)
                    else:
                        break
                    if o is op:
                        return list(sc.names)
            except Exception:  # noqa: BLE001 — UnsupportedUDF or a UDF the front end cannot read
                pass
        return _map_output_names(op.udf, names)

    def _execute(self, dry: bool = False, sink: Optional[str] = None):
        """Split the operator chain into stages and run them. Returns (python rows, column names)."""
        src = self._source
        self._last_exceptions = Counter()
        if self._join is not None:
            rows, names = _run_join(self._ctx, self._join, self._last_exceptions)
            if not self._ops:
                return rows, names
            src = self._ctx._source_from_rows(rows, names)
        elif self._parent is not None:
            rows, names = self._parent._execute()
            src = self._ctx._source_from_rows(rows, names)
        stages: List[List[Op]] = [[]]
        for op in self._ops:
            stages[-1].append(op)
            if op.kind in ("aggregate", "aggregateByKey", "unique"):
                stages.append([])
        if not stages[-1] and len(stages) > 1:
            stages.pop()
        rows = names = None
        for si, ops in enumerate(stages):
            if si > 0:
                src = self._ctx._source_from_rows(rows, names)
            last = si == len(stages) - 1
            rows, names = _run_stage(self._ctx, src, ops, self._last_exceptions,
                                     csv_sink=self._csv_sink if (sink == "csv" and last) else None)
        return rows, names


def _map_output_names(udf, names):
    """Names after a map(): a dict literal names its columns, anything else yields unnamed columns (one per tuple element)."""
    import ast as _ast
    from .frontend import get_udf_ast, _single_return
    try:
        _, body, _ = get_udf_ast(udf)
        node = body if isinstance(body, _ast.expr) else _single_return(body)
    except Exception:  # noqa: BLE001
        return [None]
    if isinstance(node, _ast.Dict) and all(isinstance(k, _ast.Constant) and isinstance(k.value, str) for k in node.keys):
        return [k.value for k in node.keys]
    if isinstance(node, _ast.Tuple):
        return [None] * len(node.elts)
    if isinstance(node, _ast.Name) and len(names) > 1:
        return list(names)  # identity-style map of the whole row
    return [None]


def csv_lazy_columns(prog, used_cols, in_types):
    """File columns the device CSV source may leave as cell references: string columns of a row stage that its prefilter
    does not read (the stage materialises them for surviving rows only). `prog` reads the projected block `used_cols`."""
    if prog.prefilter is None or prog.endpoint != C["TPLX_EP_MEMORY"]:
        return None
    early = {int(i.imm) for i in prog.prefilter.instrs if i.op == C["TPLX_OP_LDCOL"]}
    lazy = [c for k, c in enumerate(used_cols) if k not in early and in_types[c] == T_STR]
    return lazy or None


def _csv_cell(v, null_value=None) -> str:
    """Host twin of the row writer (fast_csvwriter + quoteForCSV + ryu d2fixed(8) for floats)."""
    if isinstance(v, str):
        if any(ch in v for ch in ',"\n\r'):
            return '"' + v.replace('"', '""') + '"'
        return v
    if v is None:
        return _csv_cell(null_value or "")
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, float):
        if v != v:
            return "nan"
        if v in (float("inf"), float("-inf")):
            return "Infinity" if v > 0 else "-Infinity"
        return "%.8f" % v
    return str(v)


def _row_of(cols: List[Column], values_cache: List[list], i: int):
    vals = tuple(values_cache[c][i] for c in range(len(cols)))
    return vals if len(vals) != 1 else vals[0]


def _option_cols(cols) -> List[int]:
    """Input columns that hold None values (Option[T]): the stage reads their validity bitmaps through companion columns."""
    return [c for c, col in enumerate(cols) if getattr(col, "valid", None) is not None]


def _rows_as_tuples(rows):
    return [r if isinstance(r, tuple) else (r,) for r in rows]


def _run_join(ctx, spec: JoinSpec, exc_counter: Counter):
    """A JoinOperator between two executed datasets: HashJoinStage of the reference (core/src/physical/HashJoinStage.cc; build stage
    with a hash-table endpoint + probe inside the other side's pipeline, PipelineBuilder.cc:2110-2523) on the GPU (K8,
    tplx_gpu_join_build / tplx_gpu_join_probe). Rows outside the normal case of either side (fallback rows) are joined on the
    interpreter path and merged by (probe row, build row), which is the order the normal case produces."""
    lrows, lnames = spec.left._execute()
    rrows, rnames = spec.right._execute()
    exc_counter.update(spec.left._last_exceptions)
    exc_counter.update(spec.right._last_exceptions)
    lnames = list(lnames) if lnames else []
    rnames = list(rnames) if rnames else []
    li, ri = spec.key_indices(lnames, rnames)
    names = spec.names(lnames, rnames)
    build_right = spec.build_right()
    left_outer = spec.kind == "left"
    lsrc = ctx._source_from_rows(lrows, lnames, option=True)
    rsrc = ctx._source_from_rows(rrows, rnames, option=True)
    n_left_cols, n_right_cols = len(lnames), len(rnames)

    def python_join():
        """Interpreter path of the whole join (key types the device does not hash, empty sides)."""
        L, R = _rows_as_tuples(lrows), _rows_as_tuples(rrows)
        return _py_join_pairs(L, li, R, ri, left_outer, build_right, n_right_cols), names

    if not lrows or not rrows or len(lsrc.cols) != n_left_cols or len(rsrc.cols) != n_right_cols:
        return python_join()
    lk, rk = lsrc.cols[li], rsrc.cols[ri]
    if lk.type != rk.type:  # a side whose keys are all None takes the other side's key type (NULLVALUE vs Option[T], JoinOperator.cc:121-131)
        if rk.valid is not None and not rk.present().any():
            rsrc.cols[ri] = rk = Column.from_values([None] * len(rk), lk.type)
        elif lk.valid is not None and not lk.present().any():
            lsrc.cols[li] = lk = Column.from_values([None] * len(lk), rk.type)
        else:
            raise TypeError(f"can't perform join, left column '{spec.left_col}' type {ir.TYPE_NAMES[lk.type]} is not the same as right column "
                            f"'{spec.right_col}' type {ir.TYPE_NAMES[rk.type]}")
    if lk.type == T_F64 or len(names) > C["TPLX_MAX_COLS"] - 2:
        return python_join()

    need_idx = bool(lsrc.fallback or rsrc.fallback)
    lcols, rcols = list(lsrc.cols), list(rsrc.cols)
    if need_idx:  # original row numbers travel as one more payload column per side: the merge below orders by them
        lcols.append(Column(T_I64, lsrc.orig_index if lsrc.orig_index is not None else np.arange(lsrc.n_rows, dtype=np.int64)))
        rcols.append(Column(T_I64, rsrc.orig_index if rsrc.orig_index is not None else np.arange(rsrc.n_rows, dtype=np.int64)))
    probe_cols, build_cols, pk, bk = (lcols, rcols, li, ri) if build_right else (rcols, lcols, ri, li)
    n_probe, n_build = (lsrc.n_rows, rsrc.n_rows) if build_right else (rsrc.n_rows, lsrc.n_rows)
    devs = list(getattr(ctx, "_devices", [ctx._device])) or [ctx._device]
    block_rows = ctx._block_rows
    blocks = [(lo, min(n_probe, lo + block_rows)) for lo in range(0, n_probe, block_rows)] or [(0, 0)]
    if len(blocks) < 2:
        devs = devs[:1]  # a single probe block has nothing to shard
    backend.init(sorted(set(devs)))
    from .dist import shard_range
    import threading
    mlock = threading.Lock()

    def run_shard(k: int):
        """One task per device: the table is built once per device (broadcast of the small side), the device's contiguous run of
        probe blocks goes through it in order; no exchange between devices."""
        dev = devs[k]
        bb = backend.Block.upload(dev, build_cols, n_build)
        jn = backend.Join(bb, [c.type for c in build_cols], bk)
        outs = []
        blo, bhi = shard_range(len(blocks), k, len(devs))
        for lo, hi in blocks[blo:bhi]:
            cols = [c.slice(lo, hi) for c in probe_cols] if (lo, hi) != (0, n_probe) else probe_cols
            pb = backend.Block.upload(dev, cols, hi - lo)
            res = jn.probe(pb, [c.type for c in probe_cols], pk, left_outer=left_outer, build_first=not build_right)
            info = res.info
            with mlock:
                ctx.metrics._add(info)
                ctx.metrics.join_probe_rows = getattr(ctx.metrics, "join_probe_rows", 0) + (hi - lo)
            outs.append(res.columns())
            res.free()
            pb.free()
        with mlock:
            ctx.metrics.join_build_ms = getattr(ctx.metrics, "join_build_ms", 0.0) + jn.info["build_ms"]
        jn.free()
        bb.free()
        return outs

    if len(devs) == 1:
        shard_outs = [run_shard(0)]
    else:
        shard_outs: List[Any] = [None] * len(devs)
        errs: List[BaseException] = []

        def work(k):
            try:
                shard_outs[k] = run_shard(k)
            except BaseException as e:  # noqa: BLE001
                errs.append(e)
        ths = [threading.Thread(target=work, args=(k,)) for k in range(len(devs))]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        if errs:
            raise errs[0]
    col_vals: Optional[List[list]] = None
    for outs in shard_outs:
        for oc in outs:
            vals = [c.to_values() for c in oc]
            if col_vals is None:
                col_vals = vals
            else:
                for a, b in zip(col_vals, vals):
                    a.extend(b)
    col_vals = col_vals or []
    n_out = len(col_vals[0]) if col_vals else 0
    if not need_idx:
        rows = list(zip(*col_vals)) if len(col_vals) > 1 else list(col_vals[0]) if col_vals else []
        return rows, names
    # ---- interpreter path for the fallback rows of either side, merged in (probe row, build row) order ----
    # device layout with the index columns: first side's non-key columns (its index last), key, second side's non-key columns (index last)
    n_first = (n_left_cols if build_right else n_left_cols)  # left columns always come first
    left_idx_pos = n_first - 1                    # left non-key columns are n_left_cols - 1 payloads + the index column
    right_idx_pos = len(col_vals) - 1
    lidx, ridx = col_vals[left_idx_pos], col_vals[right_idx_pos]
    keep = [i for i in range(len(col_vals)) if i not in (left_idx_pos, right_idx_pos)]
    gpu_rows = [tuple(col_vals[c][i] for c in keep) for i in range(n_out)]
    L, R = _rows_as_tuples(lrows), _rows_as_tuples(rrows)
    lfall = {i for i, _ in lsrc.fallback}
    rfall = {i for i, _ in rsrc.fallback}
    extra = _py_join_index_pairs(L, li, R, ri, lfall, rfall)
    merged = {}
    for row, l, r in zip(gpu_rows, lidx, ridx):
        merged[(l, -1 if r is None else r)] = row
    for l, r in extra:
        merged[(l, r)] = _join_row(L[l], li, R[r], ri, n_right_cols)
    if left_outer:  # a left row is emitted with None only when nothing matched it on either path
        matched = {l for (l, r) in merged if r >= 0}
        for key in [k for k in merged if k[1] < 0 and k[0] in matched]:
            del merged[key]
        for l in lfall - matched:
            if len(L[l]) > li:
                merged[(l, -1)] = _join_row(L[l], li, None, ri, n_right_cols)
    order = sorted(merged, key=(lambda k: (k[0], k[1])) if build_right else (lambda k: (k[1], k[0])))
    rows = [merged[k] for k in order]
    if len(names) == 1:
        rows = [r[0] for r in rows]
    return rows, names


def _join_row(lrow, li, rrow, ri, n_right_cols):
    rr = rrow if rrow is not None else (None,) * n_right_cols
    return tuple(v for i, v in enumerate(lrow) if i != li) + (lrow[li],) + tuple(v for i, v in enumerate(rr) if i != ri)


def _key_of(v):
    return (type(v).__name__, v)  # 1, 1.0 and True are different keys (the reference joins equal TYPES only)


def _py_join_index_pairs(L, li, R, ri, lfall, rfall):
    """(left row, right row) pairs in which at least one side is a fallback row."""
    pairs = []
    if lfall:
        table: Dict[Any, List[int]] = {}
        for j, r in enumerate(R):
            if len(r) > ri:
                table.setdefault(_key_of(r[ri]), []).append(j)
        for l in sorted(lfall):
            if len(L[l]) > li:
                pairs += [(l, j) for j in table.get(_key_of(L[l][li]), [])]
    if rfall:
        table = {}
        for j in sorted(rfall):
            if len(R[j]) > ri:
                table.setdefault(_key_of(R[j][ri]), []).append(j)
        for l, row in enumerate(L):
            if l not in lfall and len(row) > li:
                pairs += [(l, j) for j in table.get(_key_of(row[li]), [])]
    return pairs


def _py_join_pairs(L, li, R, ri, left_outer, build_right, n_right_cols):
    """The whole join on the interpreter path (same order rules as the device path)."""
    out = []
    if build_right:
        table: Dict[Any, List[int]] = {}
        for j, r in enumerate(R):
            table.setdefault(_key_of(r[ri]), []).append(j)
        for l in L:
            ms = table.get(_key_of(l[li]), [])
            out += [_join_row(l, li, R[j], ri, n_right_cols) for j in ms]
            if not ms and left_outer:
                out.append(_join_row(l, li, None, ri, n_right_cols))
    else:
        table = {}
        for i, l in enumerate(L):
            table.setdefault(_key_of(l[li]), []).append(i)
        for r in R:
            out += [_join_row(L[i], li, r, ri, n_right_cols) for i in table.get(_key_of(r[ri]), [])]
    if out and len(out[0]) == 1:
        out = [r[0] for r in out]
    return out


def _run_stage(ctx, src: Source, ops: List[Op], exc_counter: Counter, csv_sink: Optional[list] = None):
    """One TransformStage on the GPU + CPython resolve of its exception rows."""
    end = ops[-1] if ops and ops[-1].kind in ("aggregate", "aggregateByKey", "unique") else None
    row_ops = ops[:-1] if end else ops
    in_types = [c.type for c in src.cols]
    is_csv = hasattr(src, "chunks")  # csvsource.CsvSource: the device parses the file right in front of the stage
    if is_csv and not in_types:  # missing / empty file: nothing to run (python/tests/test_csv.py:66-69)
        return _run_stage_python(ctx, Source([], [], 0, None, [], 0), ops, exc_counter)
    prog = None
    try:
        sc = StageCompiler(in_types, src.names, _option_cols(src.cols))
        for op in row_ops:
            if op.resolvers or op.ignores:
                pass  # resolvers only act on the slow path
            if op.kind == "map":
                sc.add_map(op.udf, op.id)
            elif op.kind == "filter":
                sc.add_filter(op.udf, op.id)
            elif op.kind == "withColumn":
                sc.add_with_column(op.column, op.udf, op.id)
            elif op.kind == "mapColumn":
                sc.add_map_column(op.column, op.udf, op.id)
            elif op.kind == "selectColumns":
                sc.add_select(op.columns, op.id)
            elif op.kind == "renameColumn":
                sc.add_rename(op.column, op.extra, op.id)
        out_names = list(sc.names)
        need_rowidx = end is None and (bool(src.fallback) or is_csv)
        if end is None:
            if need_rowidx:
                sc.begin_op(row_ops[-1].id if row_ops else 0)
                d = sc.new_vreg(T_I64)
                sc.emit(C["TPLX_OP_LDROW"], d)
                from .frontend import Val
                sc.row.append(Val(T_I64, d))
                sc.names.append("__rowidx")
            prog = sc.finish_memory()
        elif end.kind == "aggregate":
            prog = sc.finish_aggregate(end.udf, end.extra[0], end.extra[1], end.id)
        elif end.kind == "aggregateByKey":
            prog = sc.finish_hash(end.columns, end.udf, end.extra[0], end.extra[1], end.id)
        else:
            prog = sc.finish_hash(list(range(len(sc.row))), None, None, None, end.id)
    except UnsupportedUDF as e:
        ctx._log(f"stage falls back to the CPython path: {e}")
        return _run_stage_python(ctx, src.to_host_source() if is_csv else src, ops, exc_counter)

    used_cols = list(range(len(in_types)))
    if is_csv:  # projection pushdown: the device decodes only the columns the stage loads
        used_cols = ir.referenced_inputs(prog)
        if len(used_cols) > C["TPLX_MAX_COLS"]:
            ctx._log(f"stage reads {len(used_cols)} columns (> TPLX_MAX_COLS): CPython path")
            return _run_stage_python(ctx, src.to_host_source(), ops, exc_counter)
        ir.project_inputs(prog, used_cols)
    dev = ctx._device
    backend.init(sorted(set(getattr(ctx, "_devices", [dev]))))
    stage = backend.Stage(prog)
    block_rows = ctx._block_rows
    in_values: Optional[List[list]] = None  # python values of input columns, built lazily for resolve

    csv_rows: Dict[int, Any] = {}  # CSV input: python value of the rows the interpreter path needs

    def input_row(i: int):
        nonlocal in_values
        if is_csv:
            return csv_rows[i]
        if in_values is None:
            in_values = [c.to_values() for c in src.cols]
        return _row_of(src.cols, in_values, i)

    fallback = list(src.fallback)

    n = src.n_rows
    starts = list(range(0, n, block_rows)) or [0]
    devs = list(getattr(ctx, "_devices", [dev])) or [dev]
    if is_csv or len(starts) < 2:
        devs = devs[:1]  # the CSV source parses chunk after chunk on one device; a single block has nothing to shard
    import threading
    mlock = threading.Lock()

    class Shard:
        """What one task (= one device's contiguous run of blocks, LocalBackend.cc:679-735) produced."""
        def __init__(self):
            self.out_cols: List[List[Column]] = []
            self.excs: List[np.ndarray] = []
            self.partials: List[List[int]] = []
            self.held: List[tuple] = []
            self.row_no = 0  # rows written + exceptions so far (TransformTask::_outputRowCounter)

    def fetch_cols(res, lo, rowmap):
        oc = res.columns()
        if need_rowidx:
            if rowmap is not None:
                oc[-1].data = rowmap[oc[-1].data]
            oc[-1].data += lo
        return oc

    def consume(sh: "Shard", res, lo, parse, data):
        """Take one block's result into the shard (exception records, output columns or partial aggregate)."""
        info = res.info
        with mlock:
            ctx.metrics._add(info)
        exc = res.exceptions()
        rowmap = None
        if parse is not None:
            pinfo = parse.info
            ctx.metrics.csv_rows += int(pinfo.n_rows)
            ctx.metrics.csv_bad_rows += int(pinfo.n_bad)
            ctx.metrics.csv_parse_ms += float(pinfo.parse_ms)
            if pinfo.n_bad:  # block row -> data row
                rowmap = parse.rowmap().astype(np.int64)
                raw = data.tobytes()
                for bad in parse.bad_rows():
                    fallback.append((lo + int(bad["row"]), src.line_object(raw[int(bad["line_start"]):int(bad["line_end"])], False)))
        if len(exc):
            exc = exc.copy()
            if rowmap is not None:
                exc["row"] = rowmap[exc["row"]]
            if parse is not None:  # text of the rows whose UDF raised, decoded as the device decoded them
                ends = parse.row_ends().astype(np.int64)
                ends[0] = -1 if ends[0] == 0xFFFFFFFF else ends[0]
                raw = data.tobytes()
                for r_ in exc["row"]:
                    a_ = int(ends[r_]) + 1
                    while raw[a_] in (10, 13):
                        a_ += 1
                    csv_rows[lo + int(r_)] = src.line_object(raw[a_:int(ends[r_ + 1])], True)
            exc["row"] += lo
            sh.excs.append(exc)
        if prog.endpoint == C["TPLX_EP_MEMORY"]:
            frn = sh.row_no  # the block ran with this first_row_no
            sh.row_no += int(info.n_out_rows) + int(info.n_exceptions)
            if csv_sink is not None:
                sh.held.append((res, lo, rowmap, frn, getattr(sh, "dev", dev)))  # decide at the end: device CSV writer or column fetch + merge
                return
            sh.out_cols.append(fetch_cols(res, lo, rowmap))
        elif prog.endpoint == C["TPLX_EP_AGGREGATE"]:
            sh.partials.append(res.aggregate_bits())
        res.free()

    shards: List[Shard] = []
    agg_combined: Optional[List[int]] = None
    hash_shares: List[List[Column]] = []
    if is_csv:
        sh = Shard()
        base = 0
        col_types = [t if c in used_cols else backend.CSV_SKIP for c, t in enumerate(in_types)]
        lazy = csv_lazy_columns(prog, used_cols, in_types)
        for data, skip_header in src.chunks():
            buf = backend.CsvBuffer(dev, data)
            parse = buf.parse(col_types, src.delimiter, src.quotechar, skip_header, src.null_values, lazy=lazy)
            consume(sh, stage.run(parse.block, sh.row_no), base, parse, data)
            base += int(parse.info.n_rows)
            parse.free()
            buf.free()
        src.total_rows = base
        shards.append(sh)
    else:
        # blocks are sharded contiguously over the context's devices (tuplex.gpu.devices): one task per device, its blocks in
        # order; concatenating the shards in device order preserves the input order (LocalBackend.cc:1104-1152). Map / filter
        # stages exchange nothing; aggregate endpoints combine through the C ABI's collectives when every device is distinct.
        from .dist import shard_range
        blocks = [(lo, min(n, lo + block_rows)) for lo in starts]
        phys = len(set(devs)) == len(devs) and len(devs) > 1  # distinct physical devices: NCCL communicator over them
        if phys:
            ctx._ensure_local_comm(devs)

        def run_shard(k: int) -> Shard:
            sh = Shard()
            sh.dev = devs[k]
            blo, bhi = shard_range(len(blocks), k, len(devs))
            for lo, hi in blocks[blo:bhi]:
                cols = [c.slice(lo, hi) for c in src.cols] if (lo, hi) != (0, n) else src.cols
                consume(sh, stage.run_host(devs[k], cols, hi - lo, sh.row_no), lo, None, None)
            if len(devs) > 1 and prog.endpoint == C["TPLX_EP_AGGREGATE"] and phys:
                # this device's partial = its blocks folded in block order; collective: NCCL all-gather + fold in device order
                part = None
                for p in sh.partials:
                    part = p if part is None else [_acc_bits(a.kind, _acc_combine(a.kind, _acc_value(a.kind, x), _acc_value(a.kind, y)))
                                                   for a, x, y in zip(prog.accs, part, p)]
                if part is None:
                    part = [_acc_identity_bits(a.kind) for a in prog.accs]
                sh.partials = [stage.agg_finish(devs[k], part)]
            if len(devs) > 1 and prog.endpoint == C["TPLX_EP_HASH"] and phys:
                stage.hash_exchange(devs[k])  # collective: afterwards this device's table holds the groups it owns
            return sh

        if len(devs) == 1:
            shards = [run_shard(0)]
        else:
            from concurrent.futures import ThreadPoolExecutor
            with ThreadPoolExecutor(len(devs)) as ex:
                shards = list(ex.map(run_shard, range(len(devs))))
            if prog.endpoint == C["TPLX_EP_AGGREGATE"] and phys:
                agg_combined = shards[0].partials[0]  # every device holds the same combined bits
    # one numbering over the whole stage: a shard's row numbers continue where the previous shard stopped
    out_cols_all: List[List[Column]] = []
    exc_all: List[np.ndarray] = []
    agg_partials: List[List[int]] = []
    held: List[tuple] = []
    off = 0
    for sh in shards:
        for e in sh.excs:
            if off:
                e["row_no"] += off
            exc_all.append(e)
        off += sh.row_no
        out_cols_all += sh.out_cols
        agg_partials += sh.partials
        held += sh.held
    if agg_combined is not None:
        agg_partials = [agg_combined]
    excs = np.concatenate(exc_all) if exc_all else np.zeros(0, dtype=backend.EXC_DTYPE)

    # ---- endpoints --------------------------------------------------------------------------------
    if prog.endpoint == C["TPLX_EP_MEMORY"]:
        ncols = len(prog.out_cols) - prog.hidden_out_cols
        if csv_sink is not None:
            # CSV sink: when no row took the interpreter path the rows are formatted on the device (K7) in block order
            ok = not len(excs) and not fallback and not any(prog.out_null_of)  # the device writer prints values, not None cells
            if ok:
                for res, *_ in held:
                    txt = res.csv_bytes(n_cols=ncols - (1 if need_rowidx else 0))
                    if txt is None:  # f64 output column: host formatter
                        ok = False
                        break
                    csv_sink.append(txt)
            elif len(excs) and not fallback and not is_csv and not need_rowidx and not any(prog.out_null_of):
                # exception rows: resolve them in CPython, put the resolved rows back into their slots ON THE DEVICE (K9,
                # ResolveTask::executeInOrder) and keep the device row writer
                chunks = _device_merge_csv(held, row_ops, src, input_row, [t for _, t in prog.out_cols[:ncols]], exc_counter)
                if chunks is not None:
                    csv_sink.extend(chunks)
                    ok = True
            if ok:
                for res, *_ in held:
                    res.free()
                stage.close()
                return None, out_names
            del csv_sink[:]
            for res, lo_, rowmap_, *_ in held:
                out_cols_all.append(fetch_cols(res, lo_, rowmap_))
                res.free()
        merged_vals = [sum((oc[c].to_values() for oc in out_cols_all), []) for c in range(ncols)]
        n_out = len(merged_vals[0]) if ncols else 0
        user_cols = ncols - (1 if need_rowidx else 0)
        normal_rows = [tuple(merged_vals[c][i] for c in range(user_cols)) if user_cols != 1 else merged_vals[0][i] for i in range(n_out)]
        # resolve exception rows in CPython, merge by row number (ResolveTask::executeInOrder)
        resolved: List[Tuple[int, int, Any]] = []  # (input row, row_no, value) for rows that produced output
        for e in excs:
            i = int(e["row"])
            try:
                val, _ = pyexec.run_row(row_ops, input_row(i), src.names)
                resolved.append((i, int(e["row_no"]), val))
            except Dropped:
                pass
            except Exception as ex:  # noqa: BLE001 — stays an exception, counted like the reference's exception_counts
                exc_counter[(getattr(ex, "tplx_op", int(e["op_id"])), type(ex).__name__)] += 1
        if not need_rowidx:
            rows = _merge_by_rowno(normal_rows, excs, resolved)
        else:
            # rows outside the normal-case schema run entirely on the CPython path; merge by original position
            idx_normal = merged_vals[-1]
            orig = src.orig_index
            keyed = [(int(orig[j]) if orig is not None else int(j), r) for j, r in zip(idx_normal, normal_rows)]
            keyed += [(int(orig[i]) if orig is not None else i, v) for i, _, v in resolved]
            for pos, obj in fallback:
                try:
                    val, _ = pyexec.run_row(row_ops, obj, src.names)
                    keyed.append((pos, val))
                except Dropped:
                    pass
                except Exception as ex:  # noqa: BLE001
                    exc_counter[(getattr(ex, "tplx_op", 0), type(ex).__name__)] += 1
            keyed.sort(key=lambda t: t[0])
            rows = [r for _, r in keyed]
        stage.close()
        return rows, out_names

    if prog.endpoint == C["TPLX_EP_AGGREGATE"]:
        combine, init = end.extra
        inits = list(init) if isinstance(init, (tuple, list)) else [init]
        # thread slot starts from the initial value; partials combined in block (partition) order
        # (TransformTask.cc:218-230,278-299)
        accs = list(inits)
        for part in agg_partials:
            vals = [_acc_value(a.kind, b) for a, b in zip(prog.accs, part)]
            accs = [_acc_combine(a.kind, x, y) for a, x, y in zip(prog.accs, accs, vals)]
        value = tuple(accs) if isinstance(init, (tuple, list)) else accs[0]
        # exception rows + fallback rows: fold on the CPython path with the user's own aggregate UDF
        for i in [int(e["row"]) for e in excs]:
            value = _py_fold(row_ops, end, value, input_row(i), src.names, exc_counter)
        for _, obj in fallback:
            value = _py_fold(row_ops, end, value, obj, src.names, exc_counter)
        stage.close()
        return [value], [None] * (len(value) if isinstance(value, tuple) else 1)

    # hash endpoint: every distinct device holds the groups it owns after the exchange (a single table otherwise)
    nk = prog.n_keys
    vals: List[list] = []
    for dv in (sorted(set(devs), key=devs.index) if not is_csv else [dev]):
        res = stage.hash_finish(dv)
        cols = res.columns()
        res.free()
        part_vals = [c.to_values() for c in cols]
        vals = part_vals if not vals else [a_ + b_ for a_, b_ in zip(vals, part_vals)]
    n_out = len(vals[0]) if vals else 0
    table: Dict[Any, list] = {}
    order: List[Any] = []
    for i in range(n_out):
        key = tuple(vals[c][i] for c in range(nk))
        table[key] = [vals[nk + k][i] for k in range(len(prog.accs))]
        order.append(key)
    if end.kind == "aggregateByKey" and (len(excs) or fallback):
        combine, init = end.extra
        pending = [input_row(int(e["row"])) for e in excs] + [obj for _, obj in fallback]
        for obj in pending:
            try:
                val, names2 = pyexec.run_row(row_ops, obj, src.names)
            except Dropped:
                continue
            except Exception as ex:  # noqa: BLE001
                exc_counter[(getattr(ex, "tplx_op", 0), type(ex).__name__)] += 1
                continue
            r = pyexec.Row(val if isinstance(val, tuple) else (val,), names2)
            key = tuple(r[k] for k in end.columns)
            cur = table.get(key)
            cur_v = (tuple(cur) if isinstance(init, (tuple, list)) else cur[0]) if cur is not None else init
            try:
                nv = end.udf(cur_v, r if len(r) != 1 else r[0])
            except Exception as ex:  # noqa: BLE001
                exc_counter[(end.id, type(ex).__name__)] += 1
                continue
            if cur is None:
                order.append(key)
            table[key] = list(nv) if isinstance(nv, tuple) else [nv]
    elif end.kind == "unique" and (len(excs) or fallback):
        # rows outside the normal case (other types, CSV rows with nulls / unparsable cells, rows whose UDF raised on the device)
        # are resolved by the interpreter and join the set like any other row (ResolveTask feeds the same hash sink,
        # core/src/physical/ResolveTask.cc:618-700)
        pending = [input_row(int(e["row"])) for e in excs] + [obj for _, obj in fallback]
        for obj in pending:
            try:
                val, _ = pyexec.run_row(row_ops, obj, src.names)
            except Dropped:
                continue
            except Exception as ex:  # noqa: BLE001
                exc_counter[(getattr(ex, "tplx_op", 0), type(ex).__name__)] += 1
                continue
            key = val if isinstance(val, tuple) else (val,)
            if key not in table:
                table[key] = []
                order.append(key)
    order.sort(key=_key_order)
    rows = [tuple(list(k) + table[k]) if (len(k) + len(table[k])) != 1 else k[0] for k in order]
    names = list(prog.out_names) + [None] * len(prog.accs)
    stage.close()
    return rows, names


def _acc_value(kind: int, bits: int):
    if kind in (C["TPLX_ACC_SUM_F64"], C["TPLX_ACC_MIN_F64"], C["TPLX_ACC_MAX_F64"]):
        return ir.bits_f64(bits)
    return bits - (1 << 64) if bits >= 1 << 63 else bits


def _key_order(k):
    """Deterministic order of result groups with mixed key types (None / numbers / strings, e.g. rows from the interpreter path)."""
    return tuple((0, 0) if x is None else ((1, x) if isinstance(x, (int, float)) and not isinstance(x, bool) else
                                           ((2, int(x)) if isinstance(x, bool) else (3, str(x)))) for x in k)


def _acc_bits(kind: int, v) -> int:
    if kind in (C["TPLX_ACC_SUM_F64"], C["TPLX_ACC_MIN_F64"], C["TPLX_ACC_MAX_F64"]):
        return ir.f64_bits(float(v))
    return int(v) & ((1 << 64) - 1)


def _acc_identity_bits(kind: int) -> int:
    return {C["TPLX_ACC_SUM_I64"]: 0, C["TPLX_ACC_SUM_F64"]: 0, C["TPLX_ACC_MIN_I64"]: (1 << 63) - 1, C["TPLX_ACC_MAX_I64"]: 1 << 63,
            C["TPLX_ACC_MIN_F64"]: 0x7FF0000000000000}.get(kind, 0xFFF0000000000000)


def _acc_combine(kind: int, a, b):
    if kind in (C["TPLX_ACC_SUM_I64"],):
        s = (int(a) + int(b)) & ((1 << 64) - 1)
        return s - (1 << 64) if s >= 1 << 63 else s
    if kind == C["TPLX_ACC_SUM_F64"]:
        return float(a) + float(b)
    if kind in (C["TPLX_ACC_MIN_I64"], C["TPLX_ACC_MIN_F64"]):
        return min(a, b)
    return max(a, b)


def _py_fold(row_ops, end: Op, value, obj, names, exc_counter):
    try:
        val, names2 = pyexec.run_row(row_ops, obj, names)
        # the aggregate UDF sees the row as on the device path: a Row (columns by name or index), one column as the value itself
        r = pyexec.Row(val if isinstance(val, tuple) else (val,), names2)
        return end.udf(value, r if len(r) != 1 else r[0])
    except Dropped:
        return value
    except Exception as ex:  # noqa: BLE001
        exc_counter[(getattr(ex, "tplx_op", end.id), type(ex).__name__)] += 1
        return value


def _fits_type(v, t: int) -> bool:
    if t == T_STR:
        return isinstance(v, str)
    if t == T_F64:
        return isinstance(v, float)
    if t == T_BOOL:
        return isinstance(v, bool)
    return isinstance(v, int) and not isinstance(v, bool) and -(1 << 63) <= v < (1 << 63)


def _device_merge_csv(held, row_ops, src, input_row, out_types, exc_counter: Counter) -> Optional[List[bytes]]:
    """CSV text of every held block result with its resolved exception rows merged in order on the device
    (tplx_gpu_result_merge_resolved + tplx_gpu_result_csv). None when a resolved row does not fit the stage's output schema
    (the host path then merges and formats); exception counts are only taken over on success."""
    ncols = len(out_types)
    chunks: List[bytes] = []
    counts: Counter = Counter()
    for res, lo, _rowmap, frn, dev in held:
        ex = res.exceptions()
        if not len(ex):
            txt = res.csv_bytes(n_cols=ncols)
            if txt is None:
                return None
            chunks.append(txt)
            continue
        rows, nos = [], []
        for e in ex[np.argsort(ex["row_no"], kind="stable")]:
            try:
                val, _ = pyexec.run_row(row_ops, input_row(lo + int(e["row"])), src.names)
            except Dropped:
                continue
            except Exception as err:  # noqa: BLE001 — stays an exception
                counts[(getattr(err, "tplx_op", int(e["op_id"])), type(err).__name__)] += 1
                continue
            vt = val if isinstance(val, tuple) else (val,)
            if len(vt) != ncols or not all(_fits_type(v, t) for v, t in zip(vt, out_types)):
                return None
            rows.append(vt)
            nos.append(int(e["row_no"]))
        blk = backend.Block.upload(dev, [Column.from_values([r[c] for r in rows], out_types[c]) for c in range(ncols)], len(rows))
        merged = res.merge_resolved(blk, nos, frn)
        txt = merged.csv_bytes(n_cols=ncols)
        merged.free()
        blk.free()
        if txt is None:
            return None
        chunks.append(txt)
    exc_counter.update(counts)
    return chunks


def _merge_by_rowno(normal_rows: list, excs: np.ndarray, resolved: List[Tuple[int, int, Any]]) -> list:
    """Exception k occupied slot row_no_k of the task's output stream (TransformTask.cc:885); a resolved row
    goes back to exactly that slot, an unresolved one leaves it empty."""
    if not len(excs):
        return normal_rows
    res_by_no = {no: v for _, no, v in resolved}
    out = []
    ni = 0
    pos = 0
    for no in sorted(int(x) for x in excs["row_no"]):
        while pos < no and ni < len(normal_rows):
            out.append(normal_rows[ni])
            ni += 1
            pos += 1
        if no in res_by_no:
            out.append(res_by_no[no])
        pos += 1
    out.extend(normal_rows[ni:])
    return out


def _run_stage_python(ctx, src: Source, ops: List[Op], exc_counter: Counter):
    """Whole stage on the CPython path (UDF outside the GPU op set)."""
    end = ops[-1] if ops and ops[-1].kind in ("aggregate", "aggregateByKey", "unique") else None
    row_ops = ops[:-1] if end else ops
    vals = [c.to_values() for c in src.cols]
    items: List[Tuple[int, Any]] = []
    for i in range(src.n_rows):
        pos = int(src.orig_index[i]) if src.orig_index is not None else i
        items.append((pos, _row_of(src.cols, vals, i)))
    items += list(src.fallback)
    items.sort(key=lambda t: t[0])
    out = []
    names = list(src.names)
    for _, obj in items:
        try:
            v, names = pyexec.run_row(row_ops, obj, src.names)
            out.append(v)
        except Dropped:
            pass
        except Exception as ex:  # noqa: BLE001
            exc_counter[(getattr(ex, "tplx_op", 0), type(ex).__name__)] += 1
    if end is None:
        return out, names
    if end.kind == "aggregate":
        combine, init = end.extra
        agg = end.udf if not isinstance(end.udf, str) else eval(end.udf)
        value = init
        for v in out:
            try:
                value = agg(value, v)
            except Exception as ex:  # noqa: BLE001
                exc_counter[(end.id, type(ex).__name__)] += 1
        comb = combine if not isinstance(combine, str) else eval(combine)
        value = comb(init, value)  # thread slot (initial value) combined with the task partial
        return [value], [None]
    if end.kind == "unique":
        seen = dict.fromkeys(out)
        return list(seen), names
    combine, init = end.extra
    agg = end.udf if not isinstance(end.udf, str) else eval(end.udf)
    comb = combine if not isinstance(combine, str) else eval(combine)
    table: Dict[Any, Any] = {}
    for v in out:
        r = pyexec.Row(v if isinstance(v, tuple) else (v,), names)
        key = tuple(r[k] for k in end.columns)
        table[key] = agg(table.get(key, init), r if len(r) != 1 else r[0])
    rows = []
    for key in sorted(table, key=_key_order):
        v = comb(init, table[key])  # combine at least once per group (LocalBackend.cc:2148-2217)
        rows.append(tuple(list(key) + (list(v) if isinstance(v, tuple) else [v])))
    knames = [k if isinstance(k, str) else names[k] for k in end.columns]
    return rows, knames + [None] * (len(rows[0]) - len(knames) if rows else 1)
