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

import threading
import time
import weakref
from collections import Counter
from concurrent.futures import ThreadPoolExecutor
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import backend, ir, pyexec
from .backend import Column
from .frontend import StageCompiler, UnsupportedUDF, Val
from .ir import C, T_BOOL, T_F64, T_I64, T_STR
from .pyexec import Dropped, Op

_ENDPOINTS = ("aggregate", "aggregateByKey", "unique")  # operators that end a stage
_metrics_lock = threading.Lock()  # ctx.metrics is updated from one thread per device


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

    @property
    def col_types(self) -> List[int]:
        return [c.type for c in self.cols]

    @property
    def option_cols(self) -> List[int]:
        return _option_cols(self.cols)

    def cost(self) -> int:
        return int(self.total_rows)

    def to_host_source(self) -> "Source":
        """The whole input as a host Source (stages whose UDFs are outside the GPU op set)."""
        return self


class FileSource(Source):
    """Input of a plan that is raw file bytes, parsed on one device right in front of the first stage: CSV (K6,
    csvsource.CsvSource) and text (K10, textsource.TextSource). Planning (names, types, Option columns, cost) is done on the host
    without a device; rows that the device parse hands back (bad rows) become fallback rows of the stage."""

    plan_types = False  # DataSet.types may come from the plan alone (else from the first rows)
    projects = False    # the parse decodes only the file columns a stage loads (_StagePlan.used_cols)

    def chunks(self):
        """(uint8 array, argument of `parse`) per device buffer, in row order."""
        raise NotImplementedError

    def parse(self, buf, arg, plan):
        """The chunk resident in `buf` (backend.CsvBuffer) parsed for `plan`'s program: a backend.CsvParse."""
        raise NotImplementedError

    def count(self, metrics, info):
        """Add one parse's counters to ctx.metrics."""
        raise NotImplementedError

    def bad_row_object(self, raw: bytes, bad):
        """Python object of a bad row (tplx_csv_bad_row `bad` of the chunk text `raw`) for the interpreter path."""
        raise NotImplementedError

    def row_object(self, raw: bytes, start: int, end: int):
        """Python object of the row in raw[start:end] as the device parsed it (for rows whose UDF raised on the device)."""
        raise NotImplementedError

    def to_host_source(self) -> Source:
        raise NotImplementedError


class DeviceRows:
    """Rows that pass from one operator to the next as device column blocks: the per-block results of one device (stage results,
    their K9 merges with resolved rows, join probes) or the blocks of a cached dataset, in row order, each with the visible columns
    `types` first. rows() turns them into exactly the rows the host path produces from the same results. Owned parts are freed by
    free() (a consumer takes them once); borrowed parts (a cache's blocks) belong to someone else and free() leaves them."""

    def __init__(self, parts: list, names: List[Optional[str]], types: List[int], owned: bool = True):
        self.parts, self.names, self.types, self.owned = parts, list(names), list(types), owned
        self.n_rows = sum(int(p.info.n_out_rows) for p in parts)
        self.device = parts[0].device if parts else None

    def nullable(self, c: int) -> bool:
        return any(p.validity(c) is not None for p in self.parts)

    def stats(self) -> List[Tuple[List[int], List[int]]]:
        """(None rows, strings that are not valid UTF-8) per column of every part, counted on the device (tplx_gpu_block_stats)."""
        out = []
        for p in self.parts:
            b = p.as_block(len(self.types))
            out.append(b.stats())
            b.free()
        return out

    def none_column(self) -> bool:
        """Some column is None in every row: the host path types such a column from its values, not from the stage, so a consumer
        that depends on types (a stage, a join) takes these rows on the host path."""
        if self.n_rows == 0:
            return False
        none = [sum(col) for col in zip(*(nr for nr, _ in self.stats()))]
        return any(k == self.n_rows for k in none)

    def columns(self, part) -> List[Column]:
        return [part.column(c) for c in range(len(self.types))]

    def rows(self) -> list:
        """Python rows (a value per row for one column), fetched once; the device results are released."""
        vals: List[list] = [[] for _ in self.types]
        for p in self.parts:
            for acc, col in zip(vals, self.columns(p)):
                acc.extend(col.to_values())
        self.free()
        if len(vals) == 1:
            return vals[0]
        return list(zip(*vals))

    def csv(self, null_value: str) -> Optional[List[bytes]]:
        """CSV text of every part on the device (K7); None when a part needs the host writer."""
        chunks = [p.csv_bytes(n_cols=len(self.types), null_value=null_value) for p in self.parts]
        return None if any(c is None for c in chunks) else chunks

    def free(self):
        if not self.owned:
            return
        for p in self.parts:
            p.free()
        self.parts = []


class DeviceSource(Source):
    """Input of a plan that another operator left on the device (a join's output): its parts run through the stage as blocks."""

    def __init__(self, ctx, rows: DeviceRows):
        super().__init__([], rows.names, rows.n_rows, None, [], rows.n_rows)
        self.ctx, self.rows = ctx, rows

    @property
    def col_types(self) -> List[int]:
        return list(self.rows.types)

    @property
    def option_cols(self) -> List[int]:
        return [c for c in range(len(self.rows.types)) if self.rows.nullable(c)]

    def to_host_source(self) -> Source:
        return self.ctx._source_from_rows(self.rows.rows(), self.names)


class _CachedPart:
    """One block of a cached dataset (or of re-blocked groups, which `owns` it) as a part of DeviceRows. It reads like a stage
    result; a consumer that takes it as a block gets a view (as_block), so that freeing its input leaves the block intact."""

    def __init__(self, block, types: List[int], owns: bool = False):
        self.block, self.types, self.device, self.owns = block, list(types), block.device, owns
        n = int(block.n_rows)
        nb = block.column_bytes()
        self.info = _PartInfo(n, [nb[c] - (n + 1) * 4 if t == T_STR else 0 for c, t in enumerate(self.types)])

    def as_block(self, n_cols: Optional[int] = None):
        return self.block.view()

    def column(self, c: int) -> Column:
        return self.block.column(c, self.types[c])

    def validity(self, c: int):
        return self.block.validity(c)

    def csv_bytes(self, n_cols: int = 0, null_value: Optional[str] = None):
        """None: K7 writes stage results, so DeviceRows.csv's caller writes a block's rows with the host writer."""
        return None

    def free(self):
        if self.owns:
            self.block.free()


class _PartInfo:
    def __init__(self, n_out_rows: int, out_str_bytes: List[int]):
        self.n_out_rows, self.out_str_bytes = n_out_rows, out_str_bytes


class CacheSource(DeviceSource):
    """Input of a plan that cache() keeps on the device: blocks of tuplex.gpu.blockRows rows (the host source's cut), typed as
    Context._source_from_rows types the same rows, owned by this source and freed when the last dataset that refers to it goes.
    Every read borrows them (DeviceRows with borrowed parts)."""

    def __init__(self, ctx, blocks: list, names: List[Optional[str]], types: List[int], option_cols: List[int]):
        super().__init__(ctx, DeviceRows([_CachedPart(b, types) for b in blocks], names, types, owned=False))
        self._option_cols = list(option_cols)
        self.nbytes = sum(sum(b.column_bytes()) for b in blocks) + len(option_cols) * sum((int(b.n_rows) + 31) // 32 * 4 for b in blocks)
        with _metrics_lock:
            ctx.metrics.cache_rows += self.n_rows
            ctx.metrics.cache_bytes += self.nbytes
        weakref.finalize(self, _free_cache, list(blocks), ctx.metrics, self.nbytes)

    @property
    def option_cols(self) -> List[int]:
        return list(self._option_cols)


def _free_cache(blocks: list, metrics, nbytes: int):
    for b in blocks:
        b.free()
    with _metrics_lock:
        metrics.cache_bytes -= nbytes


def _cache_flags(types: Sequence[int], none_rows: Sequence[int], invalid_utf8: Sequence[int], n_rows: int) -> List[Tuple[int, int, bool]]:
    """(tplx_concat_flags, cached type, holds None) per column of n_rows > 0 rows: Context._source_from_rows's typing restated
    from counts. A column without None is plain T (its bitmap is dropped), one with some None is Option[T], one that is None in
    every row is i64 placeholders with a clear bitmap, whatever the stage's type was. Strings that are not valid UTF-8 are
    rewritten as decode("utf-8", "replace") gives them."""
    out = []
    for t, k, bad in zip(types, none_rows, invalid_utf8):
        utf8 = backend.CONCAT_UTF8 if t == T_STR and bad else 0
        if k == n_rows:
            out.append((backend.CONCAT_ALL_NONE, T_I64, True))
        elif k == 0:
            out.append((backend.CONCAT_DROP_VALID | utf8, t, False))
        else:
            out.append((utf8, t, True))
    return out


def _cache_plan(part_rows: Sequence[int], block_rows: int) -> List[List[Tuple[int, int, int]]]:
    """The pieces (part, first row, rows) of every cached block: rows [k * block_rows, (k + 1) * block_rows) of the parts' rows
    in order, the cut _column_blocks makes over a host source of the same rows. Empty parts give no piece."""
    blocks: List[List[Tuple[int, int, int]]] = []
    cur: List[Tuple[int, int, int]] = []
    fill = 0
    for p, n in enumerate(part_rows):
        r = 0
        while r < n:
            take = min(n - r, block_rows - fill)
            cur.append((p, r, take))
            r += take
            fill += take
            if fill == block_rows:
                blocks.append(cur)
                cur, fill = [], 0
    if cur:
        blocks.append(cur)
    return blocks


def _device_cache(ctx, rows: DeviceRows, names) -> Tuple[Optional[DataSet], Optional[list]]:
    """cache() of rows that a stage or join left on the device (at least one row): per-part statistics, column flags, then one
    typed concatenation per output block, each consumed part freed as soon as its rows are copied (the peak is the data plus one
    block). (dataset over a CacheSource, None); or, when the device runs out of memory, (None, the Python rows) with what was built
    freed, for the host path."""
    ncols = len(rows.types)
    stats = rows.stats()
    none = [sum(col) for col in zip(*(nr for nr, _ in stats))]
    bad = [sum(col) for col in zip(*(iv for _, iv in stats))]
    flags = _cache_flags(rows.types, none, bad, rows.n_rows)
    sizes = [int(p.info.n_out_rows) for p in rows.parts]
    plan = _cache_plan(sizes, ctx._block_rows)
    views: Dict[int, Any] = {}
    built: list = []
    start = [0] * len(sizes)  # rows of each part already in built blocks
    freed = 0                 # parts [0, freed) are released

    def release(upto: int):
        nonlocal freed
        for p in range(freed, upto):
            v = views.pop(p, None)
            if v is not None:
                v.free()
            if rows.owned:
                rows.parts[p].free()
        freed = max(freed, upto)

    try:
        for pieces in plan:
            for p, _, _ in pieces:
                if p not in views:
                    views[p] = rows.parts[p].as_block(ncols)
            built.append(backend.Block.concat_pieces([(views[p], f, n) for p, f, n in pieces], [f for f, _, _ in flags]))
            for p, f, n in pieces:
                start[p] = f + n
            p, f, n = pieces[-1]
            release(p + 1 if f + n == sizes[p] else p)
    except backend.GpuBackendError as e:
        if e.code != backend.E_NOMEM:
            raise
        ctx._log(f"cache() falls back to host rows: {e}")
        vals: List[list] = [[] for _ in range(ncols)]
        for b in built:
            for c, (_, t, _) in enumerate(flags):
                vals[c].extend(b.column(c, t).to_values())
            b.free()
        for p in range(freed, len(sizes)):
            for c, col in enumerate(rows.columns(rows.parts[p])):
                vals[c].extend(col.to_values()[start[p]:])
        release(len(sizes))
        rows.free()
        return None, (vals[0] if ncols == 1 else list(zip(*vals)))
    release(len(sizes))
    rows.free()
    src = CacheSource(ctx, built, names, [t for _, t, _ in flags], [c for c, (_, _, opt) in enumerate(flags) if opt])
    return DataSet(ctx, src), None


def _handoff_ok(ctx) -> bool:
    """Stage and join results may stay on the device between operators: one device (a join's build side would otherwise need
    copies between devices) and None kept in the normal case (the join consumes Option columns)."""
    return len(ctx._devices) == 1 and ctx._options.get("tuplex.gpu.optionColumns", "true") == "true"


def _count_handoff(ctx, n: int):
    with _metrics_lock:
        ctx.metrics.device_handoff_rows += int(n)


def _deliver(ctx, rows: DeviceRows, names, csv_sink: Optional[list], csv_null: str, handoff: bool):
    """The last operator's rows on the device to their consumer: as they are with `handoff`, as CSV text written by K7 into
    `csv_sink` (None returned) when every part can be written there, else as Python rows."""
    if handoff:
        return rows, names
    chunks = rows.csv(csv_null) if csv_sink is not None else None
    if chunks is not None:
        _count_handoff(ctx, rows.n_rows)
        rows.free()
        csv_sink.extend(chunks)
        return None, names
    return rows.rows(), names


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
        return src.cost()

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
        """Run the pipeline and keep its rows for every later action and branch. On one device, with None kept in the normal case,
        rows that a stage or join leaves on the device stay there as owned blocks (a CacheSource), typed, cut and encoded exactly as
        the host source of the same rows would be; otherwise (and for zero rows, fallback rows, aggregate endpoints) the rows come
        to the host and become a host source. `store_specialized` is accepted for the reference's signature."""
        src = self._source
        if isinstance(src, CacheSource) and not self._ops and self._join is None and self._parent is None:
            return DataSet(self._ctx, src)
        hash_end = bool(self._ops) and self._ops[-1].kind in ("aggregateByKey", "unique")  # groups are cached on the host path
        rows, names = self._execute(handoff=_handoff_ok(self._ctx) and not hash_end)
        if isinstance(rows, DeviceRows):
            if rows.n_rows:
                ds, rows = _device_cache(self._ctx, rows, names)
                if ds is not None:
                    return ds
            else:
                rows = rows.rows()
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
        (fast_csvwriter, PipelineBuilder.cc:1550-1722): on the device (K7, tplx_gpu_result_csv_nulls, None cells as `null_value`)
        when the last stage ran there without rows from the interpreter path, else by the host twin `_csv_cell`."""
        import os
        chunks: List[bytes] = []
        rows, names = self._execute(csv_sink=chunks, csv_null=null_value or "")
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
        src = self._source
        if self._join is None and self._parent is None and src is not None and (not isinstance(src, FileSource) or src.plan_types):
            try:
                sc = _compile_row_ops(self._source, self._ops)
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
        if self._parent is None and self._source is not None and len(self._source.col_types) == len(names):
            try:
                return list(_compile_row_ops(self._source, self._ops[:self._ops.index(op) + 1]).names)
            except Exception:  # noqa: BLE001 — UnsupportedUDF or a UDF the front end cannot read
                pass
        return _map_output_names(op.udf, names)

    def _execute(self, csv_sink: Optional[list] = None, csv_null: str = "", handoff: bool = False):
        """Split the operator chain into stages and run them. Returns (python rows, column names). With `csv_sink` (a list) the
        last stage may instead write its rows there as CSV text, None cells as `csv_null`, and return (None, column names). With
        `handoff` (the consumer is a join or cache()) a last row or hash stage may instead return its results on the device, as a
        DeviceRows."""
        src = self._source
        self._last_exceptions = Counter()
        if handoff and isinstance(src, CacheSource) and not self._ops and self._parent is None:
            return src.rows, list(src.names)  # the cache's blocks, borrowed: no stage needs to copy them
        if self._join is not None:
            rows, names = _run_join(self._ctx, self._join, self._last_exceptions, handoff or csv_sink is not None or bool(self._ops))
            if isinstance(rows, DeviceRows):
                if not self._ops:
                    return _deliver(self._ctx, rows, names, csv_sink, csv_null, handoff)
                if rows.none_column():
                    rows = rows.rows()
            if not self._ops:
                return rows, names
            src = DeviceSource(self._ctx, rows) if isinstance(rows, DeviceRows) else self._ctx._source_from_rows(rows, names)
        elif self._parent is not None:
            rows, names = self._parent._execute()
            src = self._ctx._source_from_rows(rows, names)
        stages: List[List[Op]] = [[]]
        for op in self._ops:
            stages[-1].append(op)
            if op.kind in _ENDPOINTS:
                stages.append([])
        if not stages[-1] and len(stages) > 1:
            stages.pop()
        rows = names = None
        for si, ops in enumerate(stages):
            if si > 0:
                src = DeviceSource(self._ctx, _reblocked(self._ctx, rows)) if isinstance(rows, DeviceRows) else self._ctx._source_from_rows(rows, names)
            last = si == len(stages) - 1
            # a stage before the last ends in an endpoint; a hash endpoint then hands its groups to the next stage on the device
            rows, names = _run_stage(self._ctx, src, ops, self._last_exceptions, csv_sink=csv_sink if last else None, csv_null=csv_null,
                                     handoff=handoff or not last)
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


def csv_lazy_columns(prog, used_cols, in_types, option_cols=()):
    """File columns the device CSV source may leave as cell references: string columns of a row stage that its prefilter
    does not read (the stage materialises them for surviving rows only). `prog` reads the projected block `used_cols`. None for
    a stage that reads an Option column: its companions are expanded from a block of device-resident columns."""
    if prog.prefilter is None or prog.endpoint != C["TPLX_EP_MEMORY"] or any(c in option_cols for c in used_cols):
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


def _compile_row_ops(src: Source, ops: Sequence[Op]) -> StageCompiler:
    """A stage compiler over `src`'s columns fed the row operators `ops`; UnsupportedUDF for a UDF outside the GPU op set and
    for any operator that is not a row operator."""
    sc = StageCompiler(src.col_types, src.names, src.option_cols)
    for op in ops:
        _add_row_op(sc, op)
    return sc


def _add_row_op(sc: StageCompiler, op: Op):
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
    else:
        raise UnsupportedUDF(f"{op.kind} is not a row operator")


def _per_device(devs: List[int], blocks: list, fn) -> list:
    """fn(device, its blocks) for every device, each over a contiguous share of `blocks`, so that concatenating the results in
    device order keeps block order. Several devices run on one thread each, all at once (their collectives meet); the results
    come back in device order and the first error is re-raised."""
    from .dist import shard_range

    def task(k: int):
        lo, hi = shard_range(len(blocks), k, len(devs))
        return fn(devs[k], blocks[lo:hi])
    if len(devs) == 1:
        return [task(0)]
    with ThreadPoolExecutor(len(devs)) as ex:
        return list(ex.map(task, range(len(devs))))


def _rows_as_tuples(rows):
    return [r if isinstance(r, tuple) else (r,) for r in rows]


def _run_join(ctx, spec: JoinSpec, exc_counter: Counter, handoff: bool = False):
    """A JoinOperator between two executed datasets: HashJoinStage of the reference (core/src/physical/HashJoinStage.cc; build stage
    with a hash-table endpoint + probe inside the other side's pipeline, PipelineBuilder.cc:2110-2523) on the GPU (K8, _join_probes).
    A side that a stage or join left on the device (DeviceRows) is joined there, unless the host path's typing or merge decides: a
    column that is None in every row, fallback rows on a host side, key types that differ, or the interpreter path. Rows outside the
    normal case of either side (fallback rows) are joined on the interpreter path and merged by (probe row, build row), which is the
    order the normal case produces. With `handoff` the output of a join that took a side from the device stays there (DeviceRows)."""
    ok = _handoff_ok(ctx)
    left, lnames = spec.left._execute(handoff=ok)
    right, rnames = spec.right._execute(handoff=ok)
    exc_counter.update(spec.left._last_exceptions)
    exc_counter.update(spec.right._last_exceptions)
    nms = [list(lnames) if lnames else [], list(rnames) if rnames else []]
    li, ri = spec.key_indices(*nms)
    names = spec.names(*nms)
    build_right = spec.build_right()
    left_outer = spec.kind == "left"
    n_left_cols, n_right_cols = len(nms[0]), len(nms[1])
    sides = [left, right]  # DeviceRows, or Python rows with their host source in srcs
    srcs = [None if isinstance(s, DeviceRows) else ctx._source_from_rows(s, nm, option=True) for s, nm in zip(sides, nms)]

    def types(i: int) -> List[int]:
        return sides[i].types if srcs[i] is None else srcs[i].col_types

    def shaped() -> bool:
        return len(types(0)) == n_left_cols and len(types(1)) == n_right_cols

    def home():
        for i in (0, 1):
            if srcs[i] is None:
                sides[i] = sides[i].rows()
                srcs[i] = ctx._source_from_rows(sides[i], nms[i], option=True)

    def python_join():
        """Interpreter path of the whole join (key types the device does not hash, empty sides)."""
        home()
        L, R = _rows_as_tuples(sides[0]), _rows_as_tuples(sides[1])
        return _py_join_pairs(L, li, R, ri, left_outer, build_right, n_right_cols), names

    if None in srcs and (not ok or not shaped() or types(0)[li] != types(1)[ri] or any(s is not None and s.fallback for s in srcs)
                         or any(s.none_column() for s in sides if isinstance(s, DeviceRows))):
        home()
    if any(s is not None and not rows for s, rows in zip(srcs, sides)) or not shaped():
        return python_join()
    if types(0)[li] != types(1)[ri]:  # both sides are host sources here
        lk, rk = srcs[0].cols[li], srcs[1].cols[ri]
        # a side whose keys are all None takes the other side's key type (NULLVALUE vs Option[T], JoinOperator.cc:121-131)
        if rk.valid is not None and not rk.present().any():
            srcs[1].cols[ri] = Column.from_values([None] * len(rk), lk.type)
        elif lk.valid is not None and not lk.present().any():
            srcs[0].cols[li] = Column.from_values([None] * len(lk), rk.type)
        else:
            raise TypeError(f"can't perform join, left column '{spec.left_col}' type {ir.TYPE_NAMES[lk.type]} is not the same as right column "
                            f"'{spec.right_col}' type {ir.TYPE_NAMES[rk.type]}")
    if types(0)[li] == T_F64 or len(names) > C["TPLX_MAX_COLS"] - 2:
        return python_join()

    need_idx = any(s is not None and s.fallback for s in srcs)  # then both sides are host sources
    cols = [None if s is None else list(s.cols) for s in srcs]  # per host side: the columns it uploads
    if need_idx:  # original row numbers travel as one more payload column per side: the merge below orders by them
        for c, s in zip(cols, srcs):
            c.append(Column(T_I64, s.orig_index if s.orig_index is not None else np.arange(s.n_rows, dtype=np.int64)))
    col_types = [types(i) if cols[i] is None else [c.type for c in cols[i]] for i in (0, 1)]
    pi, bi = (0, 1) if build_right else (1, 0)
    pk, bk = (li, ri) if build_right else (ri, li)

    def pieces(i: int) -> list:
        """Side i's device results, or row ranges of its host columns: the build side whole, the probe side by tuplex.gpu.blockRows."""
        if cols[i] is None:
            return sides[i].parts
        n = srcs[i].n_rows
        if i == bi:
            return [(0, n)]
        return [(lo, min(n, lo + ctx._block_rows)) for lo in range(0, n, ctx._block_rows)] or [(0, 0)]

    def block(i: int, dev: int, piece):
        if cols[i] is None:
            return piece.as_block(len(col_types[i]))
        lo, hi = piece
        return backend.Block.upload(dev, cols[i] if (lo, hi) == (0, srcs[i].n_rows) else [c.slice(lo, hi) for c in cols[i]], hi - lo)

    device_out = handoff and None in srcs  # one device here (_handoff_ok)

    def task(dev: int, probe_pieces) -> list:
        """One task per device: the table is built once per device (broadcast of the small side), the device's contiguous run of
        probe blocks goes through it in order; no exchange between devices. Returns the results, or the values of their columns,
        each result fetched and freed as it comes."""
        results = _join_probes(ctx, [block(bi, dev, p) for p in pieces(bi)], col_types[bi], bk, (block(pi, dev, p) for p in probe_pieces),
                               col_types[pi], pk, left_outer, not build_right)
        if device_out:
            return list(results)
        vals: List[list] = [[] for _ in range(len(col_types[0]) + len(col_types[1]) - 1)]
        for res in results:
            for acc, col in zip(vals, res.columns()):
                acc.extend(col.to_values())
            res.free()
        return vals

    probe_pieces = pieces(pi)
    devs = ctx._devices if len(probe_pieces) > 1 else [ctx._device]  # a single probe block has nothing to shard
    backend.init(sorted(set(devs)))
    on_device = [s for s in sides if isinstance(s, DeviceRows)]
    for s in on_device:
        _count_handoff(ctx, s.n_rows)
    shard_outs = _per_device(devs, probe_pieces, task)
    for s in on_device:
        s.free()
    if device_out:
        outs = shard_outs[0]
        return DeviceRows(outs, names, outs[0].out_types() if outs else []), names
    col_vals = shard_outs[0]
    for vals in shard_outs[1:]:
        for a, b in zip(col_vals, vals):
            a.extend(b)
    n_out = len(col_vals[0])
    if not need_idx:
        return (list(zip(*col_vals)) if len(col_vals) > 1 else col_vals[0]), names
    # ---- interpreter path for the fallback rows of either side, merged in (probe row, build row) order ----
    # device layout with the index columns: first side's non-key columns (its index last), key, second side's non-key columns (index last)
    left_idx_pos = n_left_cols - 1  # left columns always come first: n_left_cols - 1 non-key payloads, then the index column
    right_idx_pos = len(col_vals) - 1
    lidx, ridx = col_vals[left_idx_pos], col_vals[right_idx_pos]
    keep = [i for i in range(len(col_vals)) if i not in (left_idx_pos, right_idx_pos)]
    gpu_rows = [tuple(col_vals[c][i] for c in keep) for i in range(n_out)]
    L, R = _rows_as_tuples(sides[0]), _rows_as_tuples(sides[1])
    lfall = {i for i, _ in srcs[0].fallback}
    rfall = {i for i, _ in srcs[1].fallback}
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


def _join_probes(ctx, build: list, build_types: List[int], build_key: int, probe, probe_types: List[int], probe_key: int,
                 left_outer: bool, build_first: bool):
    """K8 over blocks of one device: the table is built over the `build` blocks (concatenated on the device when there are several)
    and every block of `probe` is probed through it in order. Yields one backend.Result per probe block and frees every block it was
    given; the table and the build block are freed also when an error ends the join."""
    t0 = time.perf_counter()
    bb = build[0] if len(build) == 1 else backend.Block.concat(build)
    if len(build) != 1:
        ms = (time.perf_counter() - t0) * 1e3
        with _metrics_lock:
            ctx.metrics.join_concat_ms = getattr(ctx.metrics, "join_concat_ms", 0.0) + ms
            ctx.metrics.join_concat_bytes = getattr(ctx.metrics, "join_concat_bytes", 0) + sum(  # n offsets per string column of a part
                nb - 4 if t == T_STR else nb for b in build for nb, t in zip(b.column_bytes(), build_types))
        for b in build:
            b.free()
    jn = None
    try:
        jn = backend.Join(bb, build_types, build_key)
        for pb in probe:
            res = jn.probe(pb, probe_types, probe_key, left_outer=left_outer, build_first=build_first)
            with _metrics_lock:
                ctx.metrics._add(res.info)
                ctx.metrics.join_probe_rows = getattr(ctx.metrics, "join_probe_rows", 0) + pb.n_rows
            yield res
            pb.free()
        with _metrics_lock:
            ctx.metrics.join_build_ms = getattr(ctx.metrics, "join_build_ms", 0.0) + jn.info["build_ms"]
    finally:
        if jn is not None:
            jn.free()
        bb.free()


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


def _run_stage(ctx, src: Source, ops: List[Op], exc_counter: Counter, csv_sink: Optional[list] = None, csv_null: str = "",
               handoff: bool = False):
    """One TransformStage on the GPU + CPython resolve of its exception rows. With `handoff` a row stage returns its results on
    the device (DeviceRows) when they can stay there."""
    end = ops[-1] if ops and ops[-1].kind in _ENDPOINTS else None
    row_ops = ops[:-1] if end else ops
    is_file = isinstance(src, FileSource)  # the device parses the file right in front of the stage
    if is_file and not src.cols:  # missing / empty file: nothing to run (python/tests/test_csv.py:66-69)
        return _run_stage_python(Source([], [], 0, None, [], 0), ops, exc_counter)
    try:
        plan = _compile_stage(src, row_ops, end)
    except UnsupportedUDF as e:
        k = _split_point(ctx, src, row_ops)
        if k is not None:
            return _run_split(ctx, src, ops, k, exc_counter, csv_sink, csv_null, handoff)
        ctx._log(f"stage falls back to the CPython path: {e}")
        return _run_stage_python(src.to_host_source(), ops, exc_counter)
    backend.init(sorted(set(ctx._devices)))
    stage = backend.Stage(plan.prog)
    hold = csv_sink is not None or handoff
    if isinstance(src, DeviceSource):
        shards = [_device_blocks(ctx, plan, stage, src, hold)]
    else:
        shards = [_file_blocks(ctx, plan, stage, src, hold)] if is_file else _column_blocks(ctx, plan, stage, src, hold)
    st = _stitch(shards, src.fallback)
    if end is None:
        rows, names = _rows_endpoint(plan, st, src, exc_counter, csv_sink, csv_null, handoff), plan.out_names
    elif end.kind == "aggregate":
        rows, names = _aggregate_endpoint(plan, st, src.names, exc_counter)
    else:
        rows, names = _hash_endpoint(plan, stage, st, list(dict.fromkeys(sh.dev for sh in shards)), src.names, exc_counter, ctx, csv_sink,
                                     csv_null, handoff)
    stage.close()
    return rows, names


class _StagePlan:
    """A stage compiled for the device: its program, the operators it runs and the layout of its columns."""

    def __init__(self, prog, row_ops: List[Op], end: Optional[Op], out_names: List[Optional[str]], need_rowidx: bool,
                 used_cols: Optional[List[int]]):
        self.prog, self.row_ops, self.end = prog, row_ops, end
        self.out_names = out_names      # output column names, without __rowidx
        self.need_rowidx = need_rowidx  # the last output column (__rowidx) holds each row's input row number
        self.used_cols = used_cols      # CSV source: the file columns the device decodes

    def fetch_cols(self, res, lo: int, rowmap: Optional[np.ndarray]) -> List[Column]:
        """Output columns of the block whose first data row is input row `lo`, __rowidx turned into input row numbers."""
        oc = res.columns()
        if self.need_rowidx:
            if rowmap is not None:
                oc[-1].data = rowmap[oc[-1].data]
            oc[-1].data += lo
        return oc


def _compile_stage(src: Source, row_ops: List[Op], end: Optional[Op]) -> _StagePlan:
    """The stage's device program; UnsupportedUDF when it has to run on the CPython path. A row stage over input that has rows
    the device does not run (fallback rows, bad rows of a file source) also outputs the input row number of each row (__rowidx), by
    which those rows are merged back in. A CSV stage decodes only the file columns the program loads (projection pushdown)."""
    projects = isinstance(src, FileSource) and src.projects
    sc = _compile_row_ops(src, row_ops)
    out_names = list(sc.names)
    need_rowidx = end is None and (bool(src.fallback) or isinstance(src, FileSource))
    if end is None:
        if need_rowidx:
            sc.begin_op(row_ops[-1].id if row_ops else 0)
            d = sc.new_vreg(T_I64)
            sc.emit(C["TPLX_OP_LDROW"], d)
            sc.row.append(Val(T_I64, d))
            sc.names.append("__rowidx")
        prog = sc.finish_memory()
    elif end.kind == "aggregate":
        prog = sc.finish_aggregate(end.udf, end.extra[0], end.extra[1], end.id)
    elif end.kind == "aggregateByKey":
        prog = sc.finish_hash(end.columns, end.udf, end.extra[0], end.extra[1], end.id)
    else:
        prog = sc.finish_hash(list(range(len(sc.row))), None, None, None, end.id)
    used_cols = None
    if projects:
        used_cols = ir.referenced_inputs(prog)
        if len(used_cols) > C["TPLX_MAX_COLS"]:
            raise UnsupportedUDF(f"stage reads {len(used_cols)} columns (> TPLX_MAX_COLS)")
        ir.project_inputs(prog, used_cols)
    return _StagePlan(prog, row_ops, end, out_names, need_rowidx, used_cols)


class _Shard:
    """What one task (= one device's contiguous run of blocks, LocalBackend.cc:679-735) produced; after _stitch, the whole stage."""

    def __init__(self, dev: Optional[int]):
        self.dev = dev
        self.out_cols: List[List[Column]] = []
        self.excs: List[np.ndarray] = []          # exception records of each block (input row, row_no, operator id)
        self.partials: List[List[int]] = []       # partial aggregate of each block
        self.held: List[tuple] = []               # CSV sink: (result, lo, rowmap, first row_no, device) until the writer is chosen
        self.fallback: List[Tuple[int, Any]] = []  # (input row, python object) of the rows the device did not run
        self.inputs: Dict[int, Any] = {}          # input row -> python object, for the rows whose UDF raised on the device
        self.row_no = 0  # rows written + exceptions so far (TransformTask::_outputRowCounter)

    def take(self, ctx, plan: _StagePlan, res, lo: int, exc: np.ndarray, rowmap: Optional[np.ndarray], hold: bool):
        """Take one block's result: its exception records (`exc`, rows counted from the block's first data row, input row `lo`),
        then its output columns, its partial aggregate or, with `hold`, the result itself."""
        info = res.info
        with _metrics_lock:
            ctx.metrics._add(info)
        if len(exc):
            exc["row"] += lo
            self.excs.append(exc)
        if plan.prog.endpoint == C["TPLX_EP_MEMORY"]:
            first_row_no = self.row_no  # the block ran with this first_row_no
            self.row_no += int(info.n_out_rows) + int(info.n_exceptions)
            if hold:
                self.held.append((res, lo, rowmap, first_row_no, self.dev))
                return
            self.out_cols.append(plan.fetch_cols(res, lo, rowmap))
        elif plan.prog.endpoint == C["TPLX_EP_AGGREGATE"]:
            self.partials.append(res.aggregate_bits())
        res.free()

    def exceptions(self) -> np.ndarray:
        return np.concatenate(self.excs) if self.excs else np.zeros(0, dtype=backend.EXC_DTYPE)

    def interpreter_rows(self) -> list:
        """Python objects of the rows outside the normal case: rows whose UDF raised on the device, then fallback rows."""
        return [self.inputs[int(e["row"])] for e in self.exceptions()] + [obj for _, obj in self.fallback]


def _file_blocks(ctx, plan: _StagePlan, stage, src: FileSource, hold: bool) -> _Shard:
    """The block loop of a file source: one device parses chunk after chunk (K6 / K10) right in front of the stage. Bad rows
    become fallback rows; the rows whose UDF raised are decoded from their text as the device decoded them."""
    sh = _Shard(ctx._device)
    base = 0
    for data, arg in src.chunks():
        buf = backend.CsvBuffer(sh.dev, data)
        parse = src.parse(buf, arg, plan)
        res = stage.run(parse.block, sh.row_no)
        pinfo, exc, rowmap = parse.info, res.exceptions(), None
        src.count(ctx.metrics, pinfo)
        raw = data.tobytes() if (pinfo.n_bad or len(exc)) else b""
        if pinfo.n_bad:  # block row -> data row
            rowmap = parse.rowmap().astype(np.int64)
            for bad in parse.bad_rows():
                sh.fallback.append((base + int(bad["row"]), src.bad_row_object(raw, bad)))
        if len(exc):
            if rowmap is not None:
                exc["row"] = rowmap[exc["row"]]
            ends = parse.row_ends().astype(np.int64)
            ends[0] = -1 if ends[0] == 0xFFFFFFFF else ends[0]
            for r in exc["row"]:
                sh.inputs[base + int(r)] = src.row_object(raw, int(ends[r]) + 1, int(ends[r + 1]))
        sh.take(ctx, plan, res, base, exc, rowmap, hold)
        base += int(pinfo.n_rows)
        parse.free()
        buf.free()
    src.total_rows = base
    return sh


def _device_blocks(ctx, plan: _StagePlan, stage, src: DeviceSource, hold: bool) -> _Shard:
    """The block loop over rows another operator left on the device: every part runs as a block, row numbering carried on as in
    _column_blocks. Rows whose UDF raised get their input row from that part's fetched columns, for those rows only."""
    rows = src.rows
    sh = _Shard(rows.device)
    lo = 0
    for part in rows.parts:
        n = int(part.info.n_out_rows)
        res = stage.run(part.as_block(len(rows.types)), sh.row_no)
        exc = res.exceptions()
        if len(exc):
            cols = rows.columns(part)
            for r in exc["row"]:
                vals = tuple(_value_at(c, int(r)) for c in cols)
                sh.inputs[lo + int(r)] = vals if len(vals) != 1 else vals[0]
        sh.take(ctx, plan, res, lo, exc, None, hold)
        lo += n
    _count_handoff(ctx, lo)
    return sh


def _value_at(col: Column, i: int):
    """Python value of row i of a fetched column, as Column.to_values gives it."""
    if col.valid is not None and not (int(col.valid[i >> 5]) >> (i & 31)) & 1:
        return None
    if col.type == T_STR:
        return col.data[int(col.offsets[i]):int(col.offsets[i + 1])].tobytes().decode("utf-8", "replace")
    v = col.data[i].item()
    return bool(v) if col.type == T_BOOL else v


def _column_blocks(ctx, plan: _StagePlan, stage, src: Source, hold: bool) -> List[_Shard]:
    """The block loop of a column source: blocks are sharded contiguously over the context's devices (tuplex.gpu.devices), one
    task per device, its blocks in order; concatenating the shards in device order preserves the input order
    (LocalBackend.cc:1104-1152). Map / filter stages exchange nothing; aggregate endpoints combine through the C ABI's
    collectives when every device is distinct."""
    prog, n, block_rows = plan.prog, src.n_rows, ctx._block_rows
    blocks = [(lo, min(n, lo + block_rows)) for lo in range(0, n, block_rows)] or [(0, 0)]
    devs = ctx._devices if len(blocks) > 1 else [ctx._device]  # a single block has nothing to shard
    phys = len(set(devs)) == len(devs) and len(devs) > 1  # distinct physical devices: NCCL communicator over them
    if phys:
        ctx._ensure_local_comm(devs)

    def run_shard(dev: int, dev_blocks) -> _Shard:
        sh = _Shard(dev)
        for lo, hi in dev_blocks:
            cols = [c.slice(lo, hi) for c in src.cols] if (lo, hi) != (0, n) else src.cols
            res = stage.run_host(dev, cols, hi - lo, sh.row_no)
            sh.take(ctx, plan, res, lo, res.exceptions(), None, hold)
        if phys and prog.endpoint == C["TPLX_EP_AGGREGATE"]:
            # this device's partial = its blocks folded in block order; collective: NCCL all-gather + fold in device order
            part = None
            for p in sh.partials:
                part = p if part is None else [_acc_bits(a.kind, _acc_combine(a.kind, _acc_value(a.kind, x), _acc_value(a.kind, y)))
                                               for a, x, y in zip(prog.accs, part, p)]
            if part is None:
                part = [_acc_identity_bits(a.kind) for a in prog.accs]
            sh.partials = [stage.agg_finish(dev, part)]
        if phys and prog.endpoint == C["TPLX_EP_HASH"]:
            stage.hash_exchange(dev)  # collective: afterwards this device's table holds the groups it owns
        return sh

    shards = _per_device(devs, blocks, run_shard)
    if phys and prog.endpoint == C["TPLX_EP_AGGREGATE"]:
        for sh in shards[1:]:
            sh.partials = []  # every device holds the same combined bits
    if any(sh.excs for sh in shards):
        vals = [c.to_values() for c in src.cols]
        for sh in shards:
            sh.inputs = {int(i): _row_of(src.cols, vals, int(i)) for e in sh.excs for i in e["row"]}
    return shards


def _stitch(shards: List[_Shard], fallback: List[Tuple[int, Any]]) -> _Shard:
    """The shards as one record, behind the source's `fallback` rows, with one numbering over the whole stage: a shard's row
    numbers continue where the previous shard stopped."""
    st = _Shard(None)
    st.fallback = list(fallback)
    for sh in shards:
        for e in sh.excs:
            e["row_no"] += st.row_no
        st.row_no += sh.row_no
        st.out_cols += sh.out_cols
        st.excs += sh.excs
        st.partials += sh.partials
        st.held += sh.held
        st.fallback += sh.fallback
        st.inputs.update(sh.inputs)
    return st


def _rows_endpoint(plan: _StagePlan, st: _Shard, src: Source, exc_counter: Counter, csv_sink: Optional[list], csv_null: str = "",
                   handoff: bool = False):
    """Memory endpoint: the normal-case rows with the rows resolved on the CPython path merged in, in order. With a CSV sink
    the device writes the text into `csv_sink` when it can, and None is returned; with `handoff` the results stay on the device
    when they can and a DeviceRows is returned."""
    prog, row_ops = plan.prog, plan.row_ops
    ncols = len(prog.out_cols) - prog.hidden_out_cols
    user_cols = ncols - (1 if plan.need_rowidx else 0)
    excs = st.exceptions()
    if (csv_sink is not None or handoff) and not st.fallback:
        # Exception rows resolved in CPython go back into their slots ON THE DEVICE (K9, ResolveTask::executeInOrder), except when
        # they must merge with fallback rows by __rowidx. The device row writer (K7) prints None cells as `csv_null`.
        if csv_sink is not None:
            chunks = _device_merge_csv(plan, st.held, src.names, st.inputs, csv_null, exc_counter)
            if chunks is not None:
                csv_sink.extend(chunks)
                for res, *_ in st.held:
                    res.free()
                return None
        else:
            parts, counts = _device_merge(plan, st.held, src.names, st.inputs)
            if parts is not None:
                exc_counter.update(counts)
                for res, *_ in st.held:
                    if not any(p is res for p in parts):
                        res.free()
                return DeviceRows(parts, plan.out_names, [t for _, t in prog.out_cols[:user_cols]])
    for res, lo, rowmap, *_ in st.held:
        st.out_cols.append(plan.fetch_cols(res, lo, rowmap))
        res.free()
    merged_vals = [sum((oc[c].to_values() for oc in st.out_cols), []) for c in range(ncols)]
    n_out = len(merged_vals[0]) if ncols else 0
    normal_rows = [tuple(merged_vals[c][i] for c in range(user_cols)) if user_cols != 1 else merged_vals[0][i] for i in range(n_out)]
    # resolve exception rows in CPython, merge by row number (ResolveTask::executeInOrder)
    resolved: List[Tuple[int, int, Any]] = []  # (input row, row_no, value) for rows that produced output
    for e in excs:
        r = _run_py(row_ops, st.inputs[int(e["row"])], src.names, exc_counter, int(e["op_id"]))
        if r is not None:
            resolved.append((int(e["row"]), int(e["row_no"]), r[0]))
    if not plan.need_rowidx:
        return _merge_by_rowno(normal_rows, excs, resolved)
    # rows outside the normal-case schema run entirely on the CPython path; merge by original position
    orig = src.orig_index
    keyed = [(int(orig[j]) if orig is not None else int(j), r) for j, r in zip(merged_vals[-1], normal_rows)]
    keyed += [(int(orig[i]) if orig is not None else i, v) for i, _, v in resolved]
    for pos, obj in st.fallback:
        r = _run_py(row_ops, obj, src.names, exc_counter, 0)
        if r is not None:
            keyed.append((pos, r[0]))
    keyed.sort(key=lambda t: t[0])
    return [r for _, r in keyed]


def _aggregate_endpoint(plan: _StagePlan, st: _Shard, names, exc_counter: Counter):
    """Aggregate endpoint: the thread slot starts from the initial value and takes the partials in block (partition) order
    (TransformTask.cc:218-230,278-299); exception rows and fallback rows are then folded in on the CPython path with the user's
    own aggregate UDF."""
    prog, end = plan.prog, plan.end
    init = end.extra[1]
    accs = list(init) if isinstance(init, (tuple, list)) else [init]
    for part in st.partials:
        vals = [_acc_value(a.kind, b) for a, b in zip(prog.accs, part)]
        accs = [_acc_combine(a.kind, x, y) for a, x, y in zip(prog.accs, accs, vals)]
    value = tuple(accs) if isinstance(init, (tuple, list)) else accs[0]
    for obj in st.interpreter_rows():
        r = _run_py(plan.row_ops, obj, names, exc_counter, end.id)
        if r is None:
            continue
        try:
            value = end.udf(value, _endpoint_arg(*r))
        except Exception as ex:  # noqa: BLE001
            exc_counter[(end.id, type(ex).__name__)] += 1
    return [value], [None] * (len(value) if isinstance(value, tuple) else 1)


def _hash_endpoint(plan: _StagePlan, stage, st: _Shard, devs: List[int], names, exc_counter: Counter, ctx=None, csv_sink: Optional[list] = None,
                   csv_null: str = "", handoff: bool = False):
    """Hash endpoint (aggregateByKey, unique): each of `devs` holds the groups it owns after the exchange (a single table
    otherwise). Given the context: on one device, with None kept in the normal case and no row for the interpreter, the groups are ordered on the
    device (_device_groups) and stay there: with `handoff` they are returned as DeviceRows, with a CSV sink K7 writes them into
    `csv_sink` (None is returned), else they are fetched in that order. Otherwise rows outside the normal case (other types, CSV rows
    with nulls / unparsable cells, rows whose UDF raised on the device) are resolved by the interpreter and join the groups like any
    other row (ResolveTask feeds the same hash sink, core/src/physical/ResolveTask.cc:618-700), and the groups are sorted here."""
    prog, end = plan.prog, plan.end
    nk = prog.n_keys
    out_names = list(prog.out_names) + [None] * len(prog.accs)
    vals: List[list] = []
    first = None
    if ctx is not None and len(devs) == 1 and _handoff_ok(ctx) and not st.interpreter_rows():
        first = stage.hash_finish(devs[0])
        first.device = devs[0]
        groups = _device_groups(first, nk)
        if groups is not None:
            return _deliver(ctx, DeviceRows([groups], out_names, groups.out_types()), out_names, csv_sink, csv_null, handoff)
    for dv in devs:
        res = first if first is not None else stage.hash_finish(dv)
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
    init = end.extra[1] if end.kind == "aggregateByKey" else None
    for obj in st.interpreter_rows():
        r = _run_py(plan.row_ops, obj, names, exc_counter, 0)
        if r is None:
            continue
        val, row_names = r
        if end.kind == "unique":
            key = val if isinstance(val, tuple) else (val,)
            if key not in table:
                table[key] = []
                order.append(key)
            continue
        key = _group_key(val, row_names, end.columns)
        cur = table.get(key)
        cur_v = (tuple(cur) if isinstance(init, (tuple, list)) else cur[0]) if cur is not None else init
        try:
            nv = end.udf(cur_v, _endpoint_arg(val, row_names))
        except Exception as ex:  # noqa: BLE001
            exc_counter[(end.id, type(ex).__name__)] += 1
            continue
        if cur is None:
            order.append(key)
        table[key] = list(nv) if isinstance(nv, tuple) else [nv]
    order.sort(key=_key_order)
    rows = [tuple(list(k) + table[k]) if (len(k) + len(table[k])) != 1 else k[0] for k in order]
    return rows, out_names


def _device_groups(res, nk: int):
    """The groups of a hash_finish result in the host path's order (_key_order), sorted on the device by their nk key columns (K11,
    Result.sort_by_keys), and typed as Context._source_from_rows types the same rows: a column without None loses its bitmap. The
    sorted result (which frees `res`), or None (res kept) where only the host path gives the answer: no group, an f64 key, a string
    that is not valid UTF-8 (the host decodes it with "replace", and distinct byte keys may collapse), a column that is None in
    every group (typed from its values on the host path)."""
    n = int(res.info.n_out_rows)
    types = res.out_types()
    if n == 0 or any(t == T_F64 for t in types[:nk]):
        return None
    blk = res.as_block()
    none, bad = blk.stats()
    blk.free()
    if any(bad) or any(k == n for k in none):
        return None
    out = res.sort_by_keys(nk, [backend.CONCAT_DROP_VALID if k == 0 else 0 for k in none])
    res.free()
    return out


def _reblocked(ctx, rows: DeviceRows) -> DeviceRows:
    """Rows cut at multiples of tuplex.gpu.blockRows, the cut _column_blocks makes over a host source of the same rows (so that
    an f64 aggregate over them sums the same blocks); rows that fit in one block are returned as they are."""
    sizes = [int(p.info.n_out_rows) for p in rows.parts]
    plan = _cache_plan(sizes, ctx._block_rows)
    if len(plan) <= 1:
        return rows
    views = [p.as_block(len(rows.types)) for p in rows.parts]
    blocks = [backend.Block.concat_pieces([(views[p], f, k) for p, f, k in pieces]) for pieces in plan]
    for v in views:
        v.free()
    rows.free()
    return DeviceRows([_CachedPart(b, rows.types, owns=True) for b in blocks], rows.names, rows.types)


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


def _run_py(row_ops: Sequence[Op], obj, names, exc_counter: Counter, default_op: int):
    """One row through `row_ops` on the CPython path: (value, names), or None when the row was dropped or raised. A raise stays an
    exception, counted like the reference's exception_counts under the operator that raised (`default_op` when not tagged)."""
    return _counted(exc_counter, default_op, pyexec.run_row, row_ops, obj, names)


def _counted(exc_counter: Counter, default_op: int, fn, *args):
    """fn(*args), or None when it dropped the row (Dropped) or raised: a raise is counted under the operator it is tagged with."""
    try:
        return fn(*args)
    except Dropped:
        return None
    except Exception as ex:  # noqa: BLE001
        exc_counter[(getattr(ex, "tplx_op", default_op), type(ex).__name__)] += 1
        return None


def _endpoint_arg(val, names):
    """A row as an aggregate UDF sees it, the same on every path: a Row (columns by name or index), one column as the value itself."""
    r = pyexec.Row(val if isinstance(val, tuple) else (val,), names)
    return r if len(r) != 1 else r[0]


def _group_key(val, names, key_columns) -> tuple:
    r = pyexec.Row(val if isinstance(val, tuple) else (val,), names)
    return tuple(r[k] for k in key_columns)


def _fits_type(v, t: int) -> bool:
    if t == T_STR:
        return isinstance(v, str)
    if t == T_F64:
        return isinstance(v, float)
    if t == T_BOOL:
        return isinstance(v, bool)
    return isinstance(v, int) and not isinstance(v, bool) and -(1 << 63) <= v < (1 << 63)


def _device_merge(plan: _StagePlan, held, names, inputs: Dict[int, Any]):
    """(every held block result with its resolved exception rows merged in order on the device (tplx_gpu_result_merge_resolved),
    the exception counts of the resolve). A result without exception rows is its own part. (None, None) when a resolved row does
    not fit the stage's output schema: the host path then merges, and counts the exceptions itself. A stage with __rowidx gets
    each resolved row's block row there (its input row: no fallback rows, so the order of row numbers is the input order)."""
    prog = plan.prog
    ncols = len(prog.out_cols) - prog.hidden_out_cols
    user_cols = ncols - (1 if plan.need_rowidx else 0)
    out_types = [t for _, t in prog.out_cols[:ncols]]
    option_outs = {k - 1 for k in prog.out_null_of if k}
    parts: list = []
    counts: Counter = Counter()

    def give_up():
        for p in parts:
            if not any(p is res for res, *_ in held):
                p.free()
        return None, None

    for res, lo, _rowmap, frn, dev in held:
        ex = res.exceptions()
        if not len(ex):
            parts.append(res)
            continue
        rows, nos = [], []
        for e in ex[np.argsort(ex["row_no"], kind="stable")]:
            r = _run_py(plan.row_ops, inputs[lo + int(e["row"])], names, counts, int(e["op_id"]))
            if r is None:
                continue
            vt = r[0] if isinstance(r[0], tuple) else (r[0],)
            if len(vt) != user_cols or not all(_fits_type(v, t) or (v is None and c in option_outs) for c, (v, t) in enumerate(zip(vt, out_types))):
                return give_up()
            rows.append(vt + ((int(e["row"]),) if plan.need_rowidx else ()))
            nos.append(int(e["row_no"]))
        if not rows:  # nothing resolved: the result already leaves every exception's slot empty
            parts.append(res)
            continue
        blk = backend.Block.upload(dev, [Column.from_values([r[c] for r in rows], out_types[c]) for c in range(ncols)], len(rows))
        parts.append(res.merge_resolved(blk, nos, frn))
    return parts, counts


def _device_merge_csv(plan: _StagePlan, held, names, inputs: Dict[int, Any], null_value: str, exc_counter: Counter) -> Optional[List[bytes]]:
    """CSV text of every held block result with its resolved exception rows merged in order on the device (_device_merge, then
    tplx_gpu_result_csv_nulls; None cells of Option output columns are written as `null_value`). None when a resolved row does not
    fit the stage's output schema or a part needs the host writer; exception counts are only taken over on success."""
    parts, counts = _device_merge(plan, held, names, inputs)
    if parts is None:
        return None
    ncols = len(plan.prog.out_cols) - plan.prog.hidden_out_cols - (1 if plan.need_rowidx else 0)
    chunks = [p.csv_bytes(n_cols=ncols, null_value=null_value) for p in parts]
    for p in parts:
        if not any(p is res for res, *_ in held):
            p.free()
    if any(c is None for c in chunks):
        return None
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


# ---- stages split at the operators the device cannot compile -------------------------------------------------------------------
_ROW_KINDS = ("map", "filter", "withColumn", "mapColumn")


def _split_point(ctx, src: Source, row_ops: List[Op]) -> Optional[int]:
    """Where a stage that does not compile as a whole runs as device segments around one CPython operator U: the position of the
    first row operator the stage compiler rejects, fed one at a time. U's output stays on the device only on one device with None
    kept in the normal case (_handoff_ok) over a source without fallback rows, so the split is taken only there, and only when a
    device segment (the operators before U, or those after it) holds a row operator. None: the whole stage runs in CPython."""
    if not _handoff_ok(ctx) or src.fallback:
        return None
    try:
        sc = StageCompiler(src.col_types, src.names, src.option_cols)
    except UnsupportedUDF:
        return None
    for k, op in enumerate(row_ops):
        try:
            _add_row_op(sc, op)
        except UnsupportedUDF:
            if any(o.kind in _ROW_KINDS for i, o in enumerate(row_ops) if i != k):
                return k
            return None
    return None


def _run_split(ctx, src: Source, ops: List[Op], k: int, exc_counter: Counter, csv_sink: Optional[list], csv_null: str, handoff: bool):
    """A stage whose row operator ops[k] (U) only CPython runs: the operators before it run as a device stage over the source (the
    file parse included) and hand their rows over on the device; U runs in CPython (_interpreter_op); the operators after it, the
    endpoint included, run as a stage of their own over U's output, split again where they need to be. Rows, their order and
    exception counts are those of the whole stage on the CPython path."""
    op = ops[k]
    ctx._log(f"stage splits at {op.kind} operator {op.id}: its UDF runs in CPython, the operators around it on the device")
    with _metrics_lock:
        ctx.metrics.split_stages += 1
    rows, names = _run_stage(ctx, src, ops[:k], exc_counter, handoff=True)
    if isinstance(rows, DeviceRows) and rows.n_rows == 0:
        rows = rows.rows()
    rows, names = _interpreter_op(ctx, rows, names, op, exc_counter)
    rest = ops[k + 1:]
    if isinstance(rows, DeviceRows):
        if not rest:
            return _deliver(ctx, rows, names, csv_sink, csv_null, handoff)
        if rows.none_column():
            rows = rows.rows()
    if not isinstance(rows, DeviceRows):
        if not rows:
            return _run_stage_python(Source([], names, 0, None, [], 0), rest, exc_counter)
        if not rest:
            return rows, names
    nsrc = DeviceSource(ctx, _reblocked(ctx, rows)) if isinstance(rows, DeviceRows) else ctx._source_from_rows(rows, names)
    return _run_stage(ctx, nsrc, rest, exc_counter, csv_sink=csv_sink, csv_null=csv_null, handoff=handoff)


def _interpreter_op(ctx, rows, names, op: Op, exc_counter: Counter):
    """U over the rows the device segment before it produced: column-wise over device rows (_columnwise_op) where it can, else
    row by row over the fetched rows. (rows, names): DeviceRows, or Python rows."""
    if isinstance(rows, DeviceRows) and op.kind != "map":
        out = _columnwise_op(ctx, rows, op, exc_counter)
        if out is not None:
            return out, out.names
    if isinstance(rows, DeviceRows):
        rows = rows.rows()
    out = [r for r in (_run_py([op], v, names, exc_counter, op.id) for v in rows) if r is not None]
    if out:
        return [v for v, _ in out], out[-1][1]
    if op.kind == "withColumn" and op.column not in names:
        return rows[:0], list(names) + [op.column]
    return rows[:0], (_map_output_names(op.udf, names) if op.kind == "map" else list(names))


def _columnwise_op(ctx, rows: DeviceRows, op: Op, exc_counter: Counter) -> Optional[DeviceRows]:
    """A filter / withColumn / mapColumn in CPython over device rows, reading only the columns its UDF and resolvers read
    (_read_set): each row is called as the row path calls it (pyexec.call_op), the columns it does not read hold None. Dropped rows
    leave the blocks through tplx_gpu_block_select; a new column is typed as Context._source_from_rows types a column, uploaded and
    put beside the untouched device columns. None (nothing consumed, nothing counted) when the new values do not make one column
    (mixed types, an int beyond i64, None in every row) or the target column does not exist: the row path then runs U."""
    from .context import typed_column
    names, types = list(rows.names), list(rows.types)
    ncols = len(types)
    target = None
    if op.kind == "mapColumn":
        if isinstance(op.column, str):
            if op.column not in names:
                return None
            target = names.index(op.column)
        elif -ncols <= op.column < ncols:
            target = op.column % ncols
        else:
            return None
    elif op.kind == "withColumn":
        target = names.index(op.column) if op.column in names else ncols
    reads = [target] if op.kind == "mapColumn" else _read_set(op, names, ncols)

    def call(value):
        v = pyexec.call_op(op, value, names)
        return (bool(v),) if op.kind == "filter" else (v,)

    counts: Counter = Counter()
    keeps, values = [], []
    for part in rows.parts:
        n = int(part.info.n_out_rows)
        cols = {c: part.column(c).to_values() for c in reads}
        empty = [None] * n
        by_col = [cols.get(c, empty) for c in range(ncols)]
        keep = np.zeros(n, dtype=bool)
        vals = []
        for i in range(n):
            row = tuple(col[i] for col in by_col)
            r = _counted(counts, op.id, call, row if ncols != 1 else row[0])
            if r is None or (op.kind == "filter" and not r[0]):
                continue
            keep[i] = True
            vals.append(r[0])
        keeps.append(keep)
        values.append(vals)
    col = None
    if target is not None:
        col = typed_column([v for vals in values for v in vals])
        if col is None:
            return None
    exc_counter.update(counts)
    with _metrics_lock:
        ctx.metrics.interpreter_values += rows.n_rows * len(reads)
    out_names, out_types = names, types
    if target is not None:
        out_names = names + [op.column] if target == ncols else names
        out_types = types + [col.type] if target == ncols else types[:target] + [col.type] + types[target + 1:]
    parts, lo = [], 0
    for part, keep in zip(rows.parts, keeps):
        kept = int(keep.sum())
        parts.append(_spliced(part, ncols, types, keep, None if col is None else col.slice(lo, lo + kept), target, out_types))
        lo += kept
    rows.parts = []  # each part now belongs to its successor
    return DeviceRows(parts, out_names, out_types)


class _SplicedPart(_CachedPart):
    """A part whose block wraps device columns owned by `deps` (freed with it): the columns of an earlier part, with some of its
    rows selected or not, beside a column uploaded from CPython values."""

    def __init__(self, block, types: List[int], deps: list):
        super().__init__(block, types, owns=True)
        self.deps = deps

    def free(self):
        super().free()
        for d in self.deps:
            d.free()
        self.deps = []


def _spliced(part, ncols: int, types: List[int], keep: np.ndarray, col: Optional[Column], target: Optional[int], out_types: List[int]):
    """`part` with the rows `keep` marks (a select on the device only when one is dropped) and `col` at column `target` (replacing
    it, or appended when target == ncols). The part is consumed."""
    if keep.all() and col is None:
        return part
    base = part.as_block(ncols)
    deps = [part]
    if not keep.all():
        sel = base.select(backend.pack_valid(keep))
        base.free()
        part.free()
        base, deps = sel, []
    if col is None:
        return _SplicedPart(base, out_types, deps)
    up = backend.Block.upload(base.device, [col], len(col))
    cols = [base.device_column(c, types[c]) for c in range(ncols)]
    if target == ncols:
        cols.append(up.device_column(0, col.type))
    else:
        cols[target] = up.device_column(0, col.type)
    return _SplicedPart(backend.Block.wrap_device(base.device, cols, len(col)), out_types, [base, up] + deps)


def _read_set(op: Op, names: List[Optional[str]], ncols: int) -> List[int]:
    """Columns a filter's or withColumn's UDF and its resolvers read from the row (all of them where the analysis cannot tell)."""
    cols: set = set()
    for f in [op.udf] + [r for _, r in op.resolvers]:
        c = _udf_reads(f, names, ncols)
        if c is None:
            return list(range(ncols))
        cols |= c
    return sorted(cols)


def _udf_reads(udf, names: List[Optional[str]], ncols: int) -> Optional[set]:
    """The columns a UDF reads from its one row parameter: every use of the parameter must be a subscript by a constant column
    name or index (negative indices count from the end). None (every column) for a UDF of several parameters (they unpack the
    row), a row of one column (the parameter is the value), a UDF whose source is not available, and any other use of the row:
    passed on, iterated, rebound, shadowed."""
    import ast as _ast
    from .frontend import get_udf_ast
    if ncols == 1:
        return None
    try:
        params, body, _ = get_udf_ast(udf)
    except Exception:  # noqa: BLE001 — the analysis gives up, it does not fail the stage
        return None
    if len(params) != 1:
        return None
    p = params[0]
    roots = body if isinstance(body, list) else [body]
    parent = {}
    for root in roots:
        for node in _ast.walk(root):
            for ch in _ast.iter_child_nodes(node):
                parent[id(ch)] = node
    cols = set()
    for root in roots:
        for node in _ast.walk(root):
            if isinstance(node, _ast.arg) and node.arg == p:
                return None
            if not (isinstance(node, _ast.Name) and node.id == p):
                continue
            sub = parent.get(id(node))
            if not (isinstance(node.ctx, _ast.Load) and isinstance(sub, _ast.Subscript) and sub.value is node and isinstance(sub.ctx, _ast.Load)):
                return None
            c = _const_column(sub.slice, names, ncols)
            if c is None:
                return None
            cols.add(c)
    return cols


def _const_column(key, names: List[Optional[str]], ncols: int) -> Optional[int]:
    import ast as _ast
    sign = 1
    if isinstance(key, _ast.UnaryOp) and isinstance(key.op, _ast.USub):
        key, sign = key.operand, -1
    if not isinstance(key, _ast.Constant):
        return None
    v = key.value
    if isinstance(v, str) and sign == 1:
        return names.index(v) if v in names else None
    if isinstance(v, int) and not isinstance(v, bool) and -ncols <= sign * v < ncols:
        return (sign * v) % ncols
    return None


def _run_stage_python(src: Source, ops: List[Op], exc_counter: Counter):
    """Whole stage on the CPython path (UDF outside the GPU op set)."""
    end = ops[-1] if ops and ops[-1].kind in _ENDPOINTS else None
    row_ops = ops[:-1] if end else ops
    vals = [c.to_values() for c in src.cols]
    items: List[Tuple[int, Any]] = []
    for i in range(src.n_rows):
        pos = int(src.orig_index[i]) if src.orig_index is not None else i
        items.append((pos, _row_of(src.cols, vals, i)))
    items += list(src.fallback)
    items.sort(key=lambda t: t[0])
    out = [r for r in (_run_py(row_ops, obj, src.names, exc_counter, 0) for _, obj in items) if r is not None]  # (value, names)
    names = out[-1][1] if out else list(src.names)
    if end is None:
        return [v for v, _ in out], names
    if end.kind == "unique":
        return list(dict.fromkeys(v for v, _ in out)), names
    combine, init = end.extra
    agg = end.udf if not isinstance(end.udf, str) else eval(end.udf)
    comb = combine if not isinstance(combine, str) else eval(combine)
    if end.kind == "aggregate":
        value = init
        for v, row_names in out:
            try:
                value = agg(value, _endpoint_arg(v, row_names))
            except Exception as ex:  # noqa: BLE001
                exc_counter[(end.id, type(ex).__name__)] += 1
        return [comb(init, value)], [None]  # thread slot (initial value) combined with the task partial
    table: Dict[Any, Any] = {}
    for v, row_names in out:
        key = _group_key(v, row_names, end.columns)
        try:
            table[key] = agg(table.get(key, init), _endpoint_arg(v, row_names))
        except Exception as ex:  # noqa: BLE001
            exc_counter[(end.id, type(ex).__name__)] += 1
    rows = []
    for key in sorted(table, key=_key_order):
        v = comb(init, table[key])  # combine at least once per group (LocalBackend.cc:2148-2217)
        rows.append(tuple(list(key) + (list(v) if isinstance(v, tuple) else [v])))
    knames = [k if isinstance(k, str) else names[k] for k in end.columns]
    return rows, knames + [None] * (len(rows[0]) - len(knames) if rows else 1)
