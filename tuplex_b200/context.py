"""Context — mirror of tuplex.Context for the hot path
(tuplex/python/tuplex/context.py:50-365; C++ side tuplex/python/src/PythonContext.cc:126-209,823-1023).

parallelize(): majority-type inference per column, rows that do not fit become fallback rows that run on
the CPython path (PythonContext::parallelize / inferType, PythonContext.cc:823,1023; fallback rows :178-204).
csv(): host-side parse into column blocks (SURVEY.md §2 row 14: CSV parsing stays on the host).
"""
from __future__ import annotations

import csv as _csv
import glob
from collections import Counter
from typing import Any, Dict, List, Optional, Sequence

import numpy as np

from . import backend
from .backend import Column
from .dataset import DataSet, Source
from .ir import C, T_BOOL, T_F64, T_I64, T_STR

_DEFAULTS = {
    # key names follow tuplex/core/src/ContextOptions.cc:182-300
    "tuplex.backend": "gpu",
    "tuplex.partitionSize": "32MB",
    "tuplex.executorCount": "0",
    "tuplex.normalcaseThreshold": "0.9",
    "tuplex.optimizer.mergeExceptionsInOrder": "true",
    "tuplex.gpu.devices": "0",
    "tuplex.gpu.blockRows": str(16 << 20),
    # None values stay in the normal case as Option[T] columns (validity bitmaps; the device code tests the flag like the
    # reference's null-aware normal case, StageBuilder.cc:644-672); false: rows holding None take the interpreter path
    "tuplex.gpu.optionColumns": "true",
    "tuplex.webui.enable": "false",
}


def _kind(v) -> Optional[int]:
    if isinstance(v, bool):
        return T_BOOL
    if isinstance(v, int):
        return T_I64 if -(1 << 63) <= v < (1 << 63) else None
    if isinstance(v, float):
        return T_F64
    if isinstance(v, str):
        return T_STR
    return None


def column_type(values) -> Optional[int]:
    """Normal-case type of one column: the majority type of its values (PythonContext::inferType), None when no value has one
    (every value None, or outside the types a column holds)."""
    cnt = Counter(_kind(v) for v in values)
    return next((k for k, _ in cnt.most_common() if k is not None), None)


def typed_column(values: Sequence) -> Optional[Column]:
    """The values as one column typed like a column of Context._source_from_rows (Option[T] where some are None), or None where
    that source would leave rows outside the normal case: a value of another type (an int beyond i64 included), or None in
    every row."""
    t = column_type(values)
    if t is None or any(v is not None and _kind(v) != t for v in values):
        return None
    return Column.from_values(values, t)


class Metrics:
    """ctx.metrics (tuplex/python/tuplex/metrics.py; JobMetrics.h): counters of the GPU path."""

    def __init__(self):
        self.rows_in = self.rows_out = self.exceptions = 0
        self.kernel_ms = self.total_ms = 0.0
        self.kernel_launches = 0
        self.csv_rows = self.csv_bad_rows = 0  # rows the device CSV source found / handed to the interpreter path
        self.csv_parse_ms = 0.0
        self.text_rows = 0  # lines the device text source split
        self.text_parse_ms = 0.0
        self.device_handoff_rows = 0  # rows passed from one operator to the next as device blocks (join sides and outputs)
        self.cache_rows = 0   # rows cache() placed in device blocks
        self.cache_bytes = 0  # device bytes the cached datasets hold now (falls when a cache is freed)
        self.split_stages = 0        # stages that ran as device segments around operators whose UDF only CPython runs
        self.interpreter_values = 0  # values such an operator read column-wise (one per row and column its UDF reads)

    def _add(self, info):
        self.rows_in += int(info.n_in_rows)
        self.rows_out += int(info.n_out_rows)
        self.exceptions += int(info.n_exceptions)
        self.kernel_ms += float(info.kernel_ms)
        self.total_ms += float(info.total_ms)
        self.kernel_launches += int(info.kernel_launches)

    def as_dict(self):
        return dict(self.__dict__)

    def as_json(self):
        import json
        return json.dumps(self.as_dict())


class Context:
    def __init__(self, conf: Optional[Dict[str, Any]] = None, **kwargs):
        self._options: Dict[str, str] = dict(_DEFAULTS)
        for src in (conf or {}), kwargs:
            for k, v in src.items():
                k = k if k.startswith("tuplex.") else "tuplex." + k
                self._options[k] = str(v).lower() if isinstance(v, bool) else str(v)
        if self._options["tuplex.backend"] not in ("gpu",):
            raise ValueError("this build provides the gpu backend only")
        devs = [int(d) for d in str(self._options["tuplex.gpu.devices"]).replace(";", ",").split(",") if d != ""]
        self._devices = devs or [0]        # blocks of a stage are sharded contiguously over these (one task per device)
        self._device = self._devices[0]
        self._block_rows = int(self._options["tuplex.gpu.blockRows"])
        self.metrics = Metrics()
        self._messages: List[str] = []

    def _ensure_local_comm(self, devs):
        """One NCCL communicator over this context's devices, created once (tplx_gpu_comm_init_local): the aggregate endpoints'
        combine / exchange run through it inside the C ABI."""
        backend.init(devs)
        if backend.comm_info(devs[0]) is None:
            backend.comm_init_local(devs)

    def _log(self, msg: str):
        self._messages.append(msg)

    def options(self, nested=False):
        return dict(self._options)

    # ---- sources -----------------------------------------------------------------------------------
    def parallelize(self, value_list, columns=None, schema=None) -> DataSet:
        if not isinstance(value_list, (list, tuple, range)):
            raise TypeError("data must be given as a list of objects")
        value_list = list(value_list)
        src = self._source_from_rows(value_list, list(columns) if columns else None, infer=True)
        return DataSet(self, src)

    def _dataset_from_rows(self, rows, names) -> DataSet:
        return DataSet(self, self._source_from_rows(rows, names))

    def _source_from_rows(self, rows: Sequence, names: Optional[List[Optional[str]]], infer: bool = True, option: Optional[bool] = None) -> Source:
        """option: None values stay in the normal case as Option[T] columns (validity bitmap) instead of making the row a fallback
        row — the form the hash join consumes (None keys go to the null bucket, nullable payload columns are gathered with their
        bitmaps); row stages still take rows with None on the interpreter path."""
        if option is None:
            option = self._options.get("tuplex.gpu.optionColumns", "true") == "true"
        n = len(rows)
        fast = self._homogeneous_source(rows, names)
        if fast is not None:
            return fast
        # row shape: majority of (is tuple, arity)
        shapes = Counter((len(r) if isinstance(r, tuple) else -1) for r in rows)
        arity = shapes.most_common(1)[0][0] if shapes else -1
        ncols = 1 if arity == -1 else arity
        if names is not None and len(names) != ncols:
            if ncols == 1 and len(names) > 1:
                raise ValueError("number of column names does not match the data")
            names = (list(names) + [None] * ncols)[:ncols]
        names = list(names) if names is not None else [None] * ncols
        # majority type per column (PythonContext::inferType)
        col_types = []
        for c in range(ncols):
            t = column_type(r[c] if arity != -1 else r for r in rows if (len(r) if isinstance(r, tuple) else -1) == arity)
            # ints and bools mixed with floats: keep the majority, the others become fallback rows
            col_types.append(T_I64 if t is None else t)
        normal_vals: List[list] = [[] for _ in range(ncols)]
        orig: List[int] = []
        fallback = []
        for i, r in enumerate(rows):
            ok = (len(r) if isinstance(r, tuple) else -1) == arity
            if ok:
                vals = r if arity != -1 else (r,)
                ok = all(_kind(v) == t or (option and v is None) for v, t in zip(vals, col_types))
            if ok:
                for c, v in enumerate(vals):
                    normal_vals[c].append(v)
                orig.append(i)
            else:
                fallback.append((i, r))
        cols = [Column.from_values(normal_vals[c], col_types[c]) for c in range(ncols)]
        oi = None if not fallback else np.asarray(orig, dtype=np.int64)
        return Source(cols, names, len(orig), oi, fallback, n)

    def _homogeneous_source(self, rows: Sequence, names) -> Optional[Source]:
        """Fast path of parallelize for the common case — every row has the same shape and every column one primitive type
        (the reference's fastI64Parallelize / fastMixedSimpleTypeTupleTransfer, python/src/PythonContext.cc:126-209,388-520):
        type checks by set(map(type, …)) and column building by numpy instead of per-value Python code."""
        n = len(rows)
        if n == 0:
            return None
        prim = {int: T_I64, float: T_F64, str: T_STR, bool: T_BOOL}
        row_types = set(map(type, rows))
        if len(row_types) != 1:
            return None
        (rt,) = row_types
        if rt in prim:
            cols_vals = [rows]
        elif rt is tuple:
            if len(set(map(len, rows))) != 1 or len(rows[0]) == 0:
                return None
            cols_vals = list(zip(*rows))
        else:
            return None
        types = []
        for cv in cols_vals:
            ts = set(map(type, cv))
            if len(ts) != 1 or next(iter(ts)) not in prim:
                return None
            types.append(prim[next(iter(ts))])
        ncols = len(cols_vals)
        if names is not None and len(names) != ncols:
            return None  # let the general path report / pad
        names = list(names) if names is not None else [None] * ncols
        try:
            cols = [Column.from_values(cv, t) for cv, t in zip(cols_vals, types)]
        except OverflowError:
            return None  # ints beyond 64 bits take the general path (fallback rows)
        return Source(cols, names, n, None, [], n)

    def text(self, pattern, null_values=None) -> DataSet:
        """tuplex.Context.text (python/tuplex/context.py:367-387): every line of the files is one row of type str; lines equal to a
        null value become None (the column is then Option[str]). Planning reads the files on the host; the lines themselves are
        split on the GPU when the first stage runs (textsource.TextSource -> tplx_gpu_text_parse)."""
        from .textsource import text_source
        return DataSet(self, text_source(self, pattern, null_values))

    def csv(self, pattern, columns=None, header=None, delimiter=None, quotechar='"', null_values=[''], type_hints={}) -> DataSet:
        """tuplex.Context.csv (python/tuplex/context.py:203-290). Planning (delimiter, header, normal-case types) looks at
        a sample of the first file on the host, like the reference's CSVStatistic; the rows themselves are parsed on
        the GPU when the first stage runs (csvsource.CsvSource -> tplx_gpu_csv_parse)."""
        from . import csvsource as cs
        files = sorted(f for p in pattern.split(",") for f in (glob.glob(p) or [p]))
        import os
        missing = [fn for fn in files if not os.path.isfile(fn)]
        for fn in missing:  # the reference logs the missing file and yields an empty dataset (python/tests/test_csv.py:66-69)
            self._log(f"csv: no such file {fn!r}")
        arrays = [np.fromfile(fn, dtype=np.uint8) for fn in files if fn not in missing]
        arrays = [a for a in arrays if a.size] or [np.zeros(0, np.uint8)]
        sample = arrays[0][: cs.SAMPLE_BYTES].tobytes()
        if len(sample) == cs.SAMPLE_BYTES:  # keep whole lines only
            sample = sample[: max(sample.rfind(b"\n"), 0)]
        text = sample.decode("utf-8", "replace")
        delim = delimiter or _sniff_delimiter(text)
        rows = [[c.decode("utf-8", "replace") for c in cells] for cells, _, _ in cs.iter_rows(sample, ord(delim), ord(quotechar))]
        has_header = header if header is not None else (columns is None and bool(rows) and not _looks_numeric(rows[0]))
        names = rows[0] if (has_header and rows) else None
        data_rows = rows[1:] if has_header else rows
        if columns is not None:
            names = list(columns)
        ncols = len(names) if names is not None else (len(data_rows[0]) if data_rows else 0)
        names = names if names is not None else [None] * ncols
        nulls = list(null_values or [])
        types = cs.infer_types(data_rows[:10000], ncols, set(nulls), float(self._options.get("tuplex.normalcaseThreshold", 0.9)))
        for c in range(ncols):
            h = type_hints.get(c, type_hints.get(names[c])) if (c in type_hints or names[c] in type_hints) else None
            if h is not None:
                types[c] = _hint_type(h)
        return DataSet(self, cs.CsvSource(arrays, list(names), types, delim, quotechar, bool(has_header), nulls))


def _sniff_delimiter(text: str) -> str:
    """The sample's delimiter; ',' when the sample has none to find (a file of one column, like the 311 zip extract)."""
    if not text.strip():
        return ","
    try:
        return _csv.Sniffer().sniff(text[:65536], delimiters=",;|\t").delimiter
    except _csv.Error:
        return ","


def _hint_type(h) -> int:
    """A csv() type hint: int / float / bool / str, or typing.Optional of one of them (an Option[T] column, T | T_OPTION)."""
    import typing
    prim = {int: T_I64, float: T_F64, str: T_STR, bool: T_BOOL}
    if h in prim:
        return prim[h]
    args = typing.get_args(h)
    if len(args) == 2 and type(None) in args:
        inner = args[0] if args[1] is type(None) else args[1]
        if inner in prim:
            return prim[inner] | C["TPLX_T_OPTION"]
    raise TypeError(f"csv: unsupported type hint {h!r} (int, float, bool, str or typing.Optional of one of them)")


def _looks_numeric(cells) -> bool:
    return any(_cell_kind(c) in (T_I64, T_F64) for c in cells)


def _cell_kind(s: str) -> int:
    try:
        int(s)
        return T_I64
    except ValueError:
        pass
    try:
        float(s)
        return T_F64
    except ValueError:
        return T_STR
