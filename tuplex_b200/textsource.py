"""Text input of a plan: raw file bytes that the GPU splits into lines (K10, csrc/text.cuh) right in front of the first stage.

Mirrors the reference's text file input (python/tuplex/context.py:367-387 -> FileInputOperator + TextReader,
core/src/physical/TextReader.cc): one row of type str per line, lines equal to a null value are None.
  * planning (no device): the line count (the source's cost), and whether any line is null, which makes the column
    Option[str] with tuplex.gpu.optionColumns (else the null lines are fallback rows holding None). The reference makes the
    column Option whenever null values are given (FileInputOperator.cc:144-149); here it is Option only when a line really
    is null, the rule of the host reader below;
  * execution: chunk after chunk of at most MAX_CHUNK bytes, cut after a newline, on one device.

`read_lines` is the host reader Context.text used before K10 and is the contract the device follows (textops.cuh); it still
serves inputs the device does not take (no lines, every line null, more null values than K10 holds) and stages that run on
the interpreter path.
"""
from __future__ import annotations

import glob
from typing import List, Optional, Sequence

import numpy as np

from . import backend
from .backend import Column
from .dataset import FileSource, Source
from .ir import T_STR

# K10 writes at most 3 bytes per input byte (one U+FFFD per invalid byte) into 32-bit offsets: 1 GiB chunks stay below 4 GiB
MAX_CHUNK = 1 << 30
MAX_NULLS, MAX_NULL_BYTES = 8, 64  # tplx_text_desc limits


def text_files(pattern: str) -> List[str]:
    """Files of a text() pattern: comma-separated, each a glob (a pattern without a match stands for itself), sorted."""
    return sorted(f for p in pattern.split(",") for f in (glob.glob(p) or [p]))


def read_lines(files: Sequence[str], log) -> List[str]:
    """Every line of the files, in order: lines end at '\\n', one trailing '\\r' is stripped, invalid UTF-8 is replaced. A file
    that cannot be read is logged and skipped."""
    lines: List[str] = []
    for fn in files:
        try:
            with open(fn, "r", encoding="utf-8", errors="replace", newline="") as fp:
                data = fp.read()
        except OSError:
            log(f"text: no such file {fn!r}")
            continue
        part = data.split("\n")
        if part and part[-1] == "":
            part.pop()  # the newline that ends the last line does not start another one
        lines.extend(ln[:-1] if ln.endswith("\r") else ln for ln in part)
    return lines


def _line_bounds(arr: np.ndarray):
    """(start, end) arrays of the lines of one file, end after the '\\r' strip."""
    n = int(arr.size)
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    ends = np.flatnonzero(arr == 10).astype(np.int64)
    if arr[-1] != 10:
        ends = np.append(ends, n)
    starts = np.concatenate(([0], ends[:-1] + 1)).astype(np.int64)
    cr = (ends > starts) & (arr[np.maximum(ends - 1, 0)] == 13)
    return starts, ends - cr


def count_null_lines(arr: np.ndarray, nulls: Sequence[bytes]) -> int:
    """Lines of one file equal to a null value (UTF-8 bytes) after the '\\r' strip and the replacement, found exactly and
    vectorised: the replacement never shortens a line, so only lines no longer than the longest null value can match; of those,
    ASCII lines are compared as byte matrices and the others decoded one by one."""
    if not nulls:
        return 0
    starts, ends = _line_bounds(arr)
    lens = ends - starts
    cand = np.flatnonzero(lens <= max(len(v) for v in nulls))
    found = 0
    for ln in np.unique(lens[cand]):
        idx = cand[lens[cand] == ln]
        m = arr[starts[idx][:, None] + np.arange(ln)] if ln else np.zeros((len(idx), 0), np.uint8)
        ascii_rows = ~(m >= 0x80).any(axis=1)
        hit = np.zeros(len(idx), dtype=bool)
        for v in nulls:
            if len(v) == ln and v.isascii():
                hit |= ascii_rows & (m == np.frombuffer(v, dtype=np.uint8)).all(axis=1)
        null_set = set(nulls)
        for k in np.flatnonzero(~ascii_rows):
            hit[k] = m[k].tobytes().decode("utf-8", "replace").encode() in null_set
        found += int(hit.sum())
    return found


def count_lines(arr: np.ndarray) -> int:
    n = int(arr.size)
    return int(np.count_nonzero(arr == 10)) + (1 if n and arr[-1] != 10 else 0)


class _TextColumn:
    """The source's one column as planning sees it: its type, and its values through the host reader (no device)."""

    def __init__(self, src: "TextSource"):
        self.type = T_STR
        self._src = src

    def to_values(self) -> list:
        return self._src.host_rows()


class TextSource(FileSource):
    """Lazy text input: `arrays` = the bytes of the readable files, in order. `option`: some line is null and null lines are
    None in an Option[str] column; otherwise null lines (if any) are handed back by the device as fallback rows holding None."""

    plan_types = True

    def __init__(self, files: List[str], arrays: List[np.ndarray], null_values: Sequence[str], option: bool, n_lines: int, log):
        super().__init__([], [None], 0, None, [], n_lines)
        self.cols = [_TextColumn(self)]
        self.files, self.arrays = files, arrays
        self.null_values = list(null_values)
        self.option = option
        self.chunk_bytes = MAX_CHUNK
        self._log = log

    @property
    def option_cols(self) -> List[int]:
        return [0] if self.option else []

    def host_rows(self) -> list:
        nulls = self.null_values
        return [None if ln in nulls else ln for ln in read_lines(self.files, self._log)]

    def to_host_source(self) -> Source:
        rows = self.host_rows()
        vals = [r for r in rows if r is not None or self.option]
        fallback = [] if self.option else [(i, None) for i, r in enumerate(rows) if r is None]
        orig = None if not fallback else np.asarray([i for i, r in enumerate(rows) if r is not None], dtype=np.int64)
        return Source([Column.from_values(vals, T_STR)], [None], len(vals), orig, fallback, len(rows))

    def chunks(self):
        """Pieces of at most chunk_bytes, each ending after a newline (or at the end of its file)."""
        for arr in self.arrays:
            lo, n = 0, int(arr.size)
            while lo < n:
                hi = min(n, lo + self.chunk_bytes)
                if hi < n:
                    nl = np.flatnonzero(arr[lo:hi] == 10)
                    if not len(nl):
                        raise backend.GpuBackendError(f"text: a line longer than {self.chunk_bytes} bytes")
                    hi = lo + int(nl[-1]) + 1
                yield arr[lo:hi], None
                lo = hi

    def parse(self, buf, arg, plan):
        return buf.parse_text(self.null_values, self.option)

    def count(self, metrics, info):
        metrics.text_rows += int(info.n_rows)
        metrics.text_parse_ms += float(info.parse_ms)

    def bad_row_object(self, raw: bytes, bad):
        return None  # K10's only bad rows are null lines without Option columns

    def row_object(self, raw: bytes, start: int, end: int):
        if end > start and raw[end - 1] == 13:
            end -= 1
        s = raw[start:end].decode("utf-8", "replace")
        return None if s in self.null_values else s


def text_source(ctx, pattern: str, null_values: Optional[Sequence[str]]) -> Source:
    """Context.text's source: a TextSource parsed by K10, or the host reader's rows for the inputs K10 does not take (no
    lines, every line null, null values beyond its limits)."""
    nulls = list(null_values or [])
    files = text_files(pattern)
    readable, arrays = [], []
    for fn in files:
        try:
            arrays.append(np.fromfile(fn, dtype=np.uint8))
            readable.append(fn)
        except OSError:
            ctx._log(f"text: no such file {fn!r}")
    enc = [v.encode() for v in nulls]
    n_lines = sum(count_lines(a) for a in arrays)
    n_null = sum(count_null_lines(a, enc) for a in arrays)
    if n_lines == 0 or n_null == n_lines or len(nulls) > MAX_NULLS or sum(map(len, enc)) > MAX_NULL_BYTES:
        rows = [None if ln in nulls else ln for ln in read_lines(readable, ctx._log)]
        return ctx._source_from_rows(rows, None)
    option = n_null > 0 and ctx._options.get("tuplex.gpu.optionColumns", "true") == "true"
    return TextSource(readable, arrays, nulls, option, n_lines, ctx._log)
