"""CSV input of a plan: raw file bytes that the GPU parses (K6, csrc/csv.cuh) right in front of the first stage.

Mirrors the reference's file input operator + CSV source task:
  * planning: delimiter / header / per-column normal-case type from a sample (FileInputOperator + CSVStatistic,
    tuplex/core/src/logical/FileInputOperator.cc, utils/src/CSVUtils.cc) — done here on the host from the first
    SAMPLE_BYTES of the file, type hints win;
  * execution: projection pushdown (only the columns the stage loads are decoded, StageBuilder.cc:1045-1070), rows that
    do not fit the normal case go to the interpreter path as string cells that are re-parsed there the way the reference's
    generated Python does (PythonPipelineBuilder.cc:253-287 `parse`, :290-350 `cellInput`).

Everything in this module that touches row data on the host belongs to that interpreter path (the reference resolves
such rows in CPython too) or to planning; the normal-case parse happens on the device.
"""
from __future__ import annotations

import json
from collections import Counter
from fractions import Fraction
from typing import Any, List, Optional, Sequence

import numpy as np

from . import backend
from .backend import Column
from .dataset import FileSource, Source, csv_lazy_columns
from .ir import C, T_BOOL, T_F64, T_I64, T_STR

T_OPTION = C["TPLX_T_OPTION"]  # type flag of an Option[T] column (col_types of the device CSV source)

SAMPLE_BYTES = 1 << 20
MAX_CHUNK = 0xFFFFFFFF - (1 << 20)  # tplx_gpu_csv_upload takes < 4 GiB
_WS = " \t\n\r\x0b\x0c"
_BOOL = {"true": True, "t": True, "yes": True, "y": True, "false": False, "f": False, "no": False, "n": False}


# ---- row machine (csvmonkey.h:523-672) for the host side: sampling and interpreter-path rows -----------------
def _machine(buf: bytes, p: int, n: int, delim: int, quote: int):
    """Row starting at p in buf (buf[n] == 10 appended). Returns (cells, end) or (None, None) on underrun."""
    cells: List[bytes] = []
    qb = bytes([quote])
    while True:
        c = buf[p]
        if c in (10, 13):
            cells.append(b"")
            return cells, p
        if c == quote:
            p += 1
            b = p
            esc = False
            while True:
                q = buf.find(qb, p)
                if q < 0 or q >= n:
                    return None, None  # input ends inside a quoted cell: csvmonkey yields no row
                p = q + 1
                c = buf[p]
                if c == delim or c in (10, 13):
                    raw = buf[b:q]
                    cells.append(_dequote(raw, quote) if esc else raw)
                    break
                esc = True
                p += 1
            if c in (10, 13):
                return cells, p
            p += 1
        else:
            b = p
            while buf[p] != delim and buf[p] not in (10, 13):
                p += 1
            cells.append(buf[b:p])
            if buf[p] != delim:
                return cells, p
            p += 1


def split_line(line: bytes, delim: int, quote: int) -> List[bytes]:
    cells, _ = _machine(line + b"\n", 0, len(line), delim, quote)
    return cells if cells is not None else []


def iter_rows(data: bytes, delim: int, quote: int):
    """(cells, line_start, line_end) of every row of a buffer, sequentially (host twin of csv_find_rows_sequential)."""
    n = len(data)
    buf = data + b"\n"
    p = 0
    while True:
        while p <= n and buf[p] in (10, 13):
            p += 1
        if p > n:
            return
        cells, e = _machine(buf, p, n, delim, quote)
        if cells is None:
            return
        yield cells, p, e
        p = e + 1


def _dequote(raw: bytes, quote: int) -> bytes:
    out = bytearray()
    i = 0
    while i < len(raw):
        if raw[i] == quote:
            i += 1
            if i >= len(raw):
                break
        out.append(raw[i])
        i += 1
    return bytes(out)


def _text(b: bytes) -> str:
    return b.decode("utf-8", "replace")


# ---- typed decoders restated for the interpreter path (StringUtils.cc:22-255 behind Runtime.cc:319-385) ---------
def atoi64(s: str) -> Optional[int]:
    t = s.strip(_WS)
    if not t:
        return None
    neg = t[0] == "-"
    d = t[1:] if neg else t
    if not all("0" <= ch <= "9" for ch in d):
        return None
    x = int(d) if d else 0
    x = (-x if neg else x) & ((1 << 64) - 1)
    return x - (1 << 64) if x >= 1 << 63 else x


def atod(s: str) -> Optional[float]:
    t = s.strip(_WS)
    if not t:
        return None
    n = len(t)
    ch = lambda k: t[k] if k < n else "\0"
    p = 0
    sign = 1.0
    if ch(p) == "-":
        sign, p = -1.0, 1
    elif ch(p) == "+":
        p = 1
    value = 0.0
    while "0" <= ch(p) <= "9":
        value = 10.0 * value + (ord(ch(p)) - 48)
        p += 1
    if ch(p) == ".":
        pow10 = 10.0
        p += 1
        while "0" <= ch(p) <= "9":
            value += (ord(ch(p)) - 48) / pow10
            pow10 *= 10.0
            p += 1
    frac, scale = False, 1.0
    if ch(p) in "eE":
        p += 1
        if ch(p) == "-":
            frac, p = True, p + 1
        elif ch(p) == "+":
            p += 1
        ex = 0
        while "0" <= ch(p) <= "9":
            ex = (ex * 10 + ord(ch(p)) - 48) & 0xFFFFFFFF
            p += 1
        ex = min(ex, 308)
        while ex >= 50:
            scale *= 1e50
            ex -= 50
        while ex >= 8:
            scale *= 1e8
            ex -= 8
        while ex > 0:
            scale *= 10.0
            ex -= 1
    nanm = infm = 0
    if p == 0:
        while nanm < 3 and ch(p).lower() == "nan"[nanm] and ch(p) != "\0":
            p += 1
            nanm += 1
    if p == 0:
        while infm < 8 and ch(p).lower() == "infinity"[infm] and ch(p) != "\0":
            p += 1
            infm += 1
    if p != n:
        return None
    if nanm == 3:
        return float("nan")
    if infm in (3, 8):
        return float("inf")
    return sign * (value / scale if frac else value * scale)


def atob(s: str) -> Optional[bool]:
    return _BOOL.get(s.lower()) if 1 <= len(s) <= 5 else None


def parse_general(s: str, nulls) -> Any:
    """`parse(s)` of the reference's generated fallback code (PythonPipelineBuilder.cc:253-287)."""
    if s in nulls:
        return None
    t = s.strip()
    if t.lower() in _BOOL:
        return _BOOL[t.lower()]
    for conv in (int, float, json.loads):
        try:
            return conv(t)
        except Exception:  # noqa: BLE001
            pass
    return s


def decode_typed(cells: Sequence[bytes], types: Sequence[int], option_cols=(), nulls=()) -> tuple:
    """Cells as the device decodes them; a null cell of an Option column is None. None also marks a cell that does not convert."""
    out = []
    for k, (c, t) in enumerate(zip(cells, types)):
        s = _text(c)
        if k in option_cols and s in nulls:
            out.append(None)
            continue
        out.append(s if t == T_STR else atoi64(s) if t == T_I64 else atod(s) if t == T_F64 else atob(s))
    return tuple(out)


def _cell_kind(s: str) -> int:
    if atob(s) is not None:
        return T_BOOL
    if atoi64(s) is not None and s.strip(_WS) not in ("-",):
        return T_I64
    if atod(s) is not None:
        return T_F64
    return T_STR


def infer_types(rows: List[List[str]], ncols: int, nulls, threshold: float = 0.9) -> List[int]:
    """Majority type per column over the sample; mixed int/float columns become f64 (CSVStatistic's normal case). A column
    whose null fraction over the sample's data rows exceeds 1 - threshold is Option[T] (T | T_OPTION), and Option[str] when
    every cell is null (CSVStatistic::estimate with disableNullColumns, utils/src/CSVStatistic.cc:109-140). The comparison is
    exact, so a column with at most 10 % nulls at threshold 0.9 keeps T."""
    types = []
    band = 1 - Fraction(str(threshold))
    for c in range(ncols):
        cells = [r[c] for r in rows if len(r) == ncols]
        cnt = Counter(_cell_kind(s) for s in cells if s not in nulls)
        tot = sum(cnt.values())
        if not tot:
            t = T_STR
        elif cnt.get(T_I64, 0) >= threshold * tot:
            t = T_I64
        elif cnt.get(T_I64, 0) + cnt.get(T_F64, 0) >= threshold * tot:
            t = T_F64
        elif cnt.get(T_BOOL, 0) >= threshold * tot:
            t = T_BOOL
        else:
            t = T_STR
        if cells and Fraction(len(cells) - tot, len(cells)) > band:
            t |= T_OPTION
        types.append(t)
    return types


class _TypeOnly:
    def __init__(self, t):
        self.type = t


class CsvChunk:
    def __init__(self, data: np.ndarray, skip_header: bool, base: int):
        self.data, self.skip_header, self.base = data, skip_header, base


class CsvSource(FileSource):
    """Lazy CSV input: `files` = uint8 arrays (one per file, header row still inside when `header`). `types` may carry T_OPTION:
    such a column is Option[T], its null cells are None in the normal case."""

    projects = True

    def __init__(self, files: List[np.ndarray], names: List[Optional[str]], types: List[int], delimiter: str, quotechar: str,
                 header: bool, null_values: Sequence[str]):
        base = [t & ~T_OPTION for t in types]
        super().__init__([_TypeOnly(t) for t in base], names, 0, None, [], 0)
        self.files, self.types = files, base
        self._option_cols = [c for c, t in enumerate(types) if t & T_OPTION]
        self.delimiter, self.quotechar, self.header = delimiter, quotechar, header
        self.null_values = list(null_values)

    @property
    def option_cols(self) -> List[int]:
        return self._option_cols

    # -- chunks of at most MAX_CHUNK bytes, cut at a newline outside quotes (quote parity, like the device) ----------
    def chunks(self):
        q = ord(self.quotechar)
        for arr in self.files:
            lo, first = 0, True
            n = int(arr.size)
            while lo < n or (first and n == 0):
                hi = min(n, lo + MAX_CHUNK)
                if hi < n:
                    par = int(np.count_nonzero(arr[lo:hi] == q)) & 1
                    k = hi
                    while k > lo:  # walk back to a newline at even quote parity
                        k -= 1
                        c = arr[k]
                        if c == q:
                            par ^= 1
                        elif c in (10, 13) and par == 0:
                            break
                    if k <= lo:
                        raise backend.GpuBackendError("csv: no row boundary found inside a 4 GiB window")
                    hi = k + 1
                yield arr[lo:hi], (self.header and first)
                first = False
                lo = hi
                if n == 0:
                    break

    def cost(self) -> int:
        """Data rows = line ends of the files (the reference estimates from a sample)."""
        return int(sum(int(np.count_nonzero(a == 10)) for a in self.files))

    def parse(self, buf, skip_header: bool, plan):
        """K6 over one chunk: only the file columns the stage's program loads are decoded (projection pushdown)."""
        opt = self.option_cols
        col_types = [(t | (T_OPTION if c in opt else 0)) if c in plan.used_cols else backend.CSV_SKIP for c, t in enumerate(self.types)]
        lazy = csv_lazy_columns(plan.prog, plan.used_cols, self.types, opt)
        return buf.parse(col_types, self.delimiter, self.quotechar, skip_header, self.null_values, lazy=lazy)

    def count(self, metrics, info):
        metrics.csv_rows += int(info.n_rows)
        metrics.csv_bad_rows += int(info.n_bad)
        metrics.csv_parse_ms += float(info.parse_ms)

    def bad_row_object(self, raw: bytes, bad):
        return self.line_object(raw[int(bad["line_start"]):int(bad["line_end"])], False)

    def row_object(self, raw: bytes, start: int, end: int):
        while raw[start] in (10, 13):  # newlines between rows belong to no row
            start += 1
        return self.line_object(raw[start:end], True)

    def line_object(self, line: bytes, typed: bool):
        """Python value of one row for the interpreter path: typed=True for rows that parsed on the device (values as
        the device decoded them, None for the null cells of Option columns), False for rows that did not (every cell
        through `parse`)."""
        cells = split_line(line, ord(self.delimiter), ord(self.quotechar))
        if typed and len(cells) == len(self.types):
            vals = decode_typed(cells, self.types, self.option_cols, self.null_values)
        else:
            vals = tuple(parse_general(_text(c), self.null_values) for c in cells)
        return vals if len(vals) != 1 else vals[0]

    def _normal_case(self, cells, vals) -> bool:
        """Does a decoded row fit the normal case: every null cell in an Option column, every other cell converted."""
        return all((k in self.option_cols) if _text(c) in self.null_values else v is not None
                   for k, (c, v) in enumerate(zip(cells, vals)))

    def to_host_source(self) -> Source:
        """Whole input through the interpreter-path decoders (used when a stage's UDFs are outside the GPU op set). Null cells
        of Option columns stay in the normal case as None (validity bitmaps)."""
        normal: List[list] = [[] for _ in self.types]
        orig, fallback = [], []
        i = 0
        d, q = ord(self.delimiter), ord(self.quotechar)
        for data, skip in self.chunks():
            raw = data.tobytes()
            for k, (cells, ls, le) in enumerate(iter_rows(raw, d, q)):
                if skip and k == 0:
                    continue
                vals = decode_typed(cells, self.types, self.option_cols, self.null_values) if len(cells) == len(self.types) else None
                if vals is None or not self._normal_case(cells, vals):
                    fallback.append((i, self.line_object(raw[ls:le], False)))
                else:
                    for c, v in enumerate(vals):
                        normal[c].append(v)
                    orig.append(i)
                i += 1
        cols = [Column.from_values(normal[c], self.types[c]) for c in range(len(self.types))]
        return Source(cols, list(self.names), len(orig), None if not fallback else np.asarray(orig, dtype=np.int64), fallback, i)
