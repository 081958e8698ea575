"""The row-format boundary (K5 both ways, csrc/rowfmt.cuh; the partition split; the K2 exception partition) against a plain serializer.

The reference below restates the reference's row format from its sources, not from oracle/tplx_oracle.c:
  row       = [bitmap of the Option fields][one 8-byte slot per field][8 B var-len total iff the schema has a str field][payload]
              (Serializer.cc:1016-1117, bitmap :1041-1059 and calcBitmapSize :29-41)
  str slot  = offset from the slot's own address | size incl. the NUL << 32 (FlattenedTuple.cc:798-835)
  partition = int64 numRows, then rows back to back, split like rowToMemorySink (TransformTask.h:47-92), capacity = size - 8
              (Partition.h:161)
  exception = int64 numRows, then [rowNo, ecCode, opID, size, input row] per record (IExceptionableTask.h:22-36)
A None string field comes in three forms, all of which K5 reads:
  "empty"     "" of size 0, slot = offset | 0 (a None produced by a UDF, FlattenedTuple.cc:628). K5 writes this form.
  "zero_slot" Serializer.cc:313-338 writes no bytes for a None string and fills the slots only when the row has var-len bytes at
              all (:1071), so in a row whose string fields are all None those slots stay 0.
  "payload"   the compiled CSV path sets only `isnull` for a null cell (FlattenedTuple.cc:1255-1293); the string keeps the cell's
              text, so the slot has its size and the text is in the payload and in the var-len total ("N/A\\0": size 4).
Columns are compared as raw data: the bits of fixed-width values, string bytes and offsets, validity words with their tail bits."""
import ctypes as ct
import re
import struct
import time

import numpy as np
import pytest

from oracle import pyoracle as po
from tuplex_b200 import backend, frontend
from tuplex_b200.backend import Column, pack_valid, unpack_valid
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR

M64 = (1 << 64) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
FORMS = ("empty", "zero_slot", "payload")
E_BADARG, E_OVERFLOW = -4, -7


# ---- the reference, restated ------------------------------------------------------------------------------------------------
def f64_bits(v):
    return struct.unpack("<Q", struct.pack("<d", v))[0]


def bits_f64(b):
    return struct.unpack("<d", struct.pack("<Q", b & M64))[0]


def _fixed_slot(t, v):
    return f64_bits(v) if t == T_F64 else int(v) & M64  # bool: an i64 0 / 1


def serialize_row(values, schema, none_str="empty", none_num=0, null_text=b"N/A"):
    """One row. schema: [(type, is_option)]; values: int / float / bool / bytes / None. none_str: the form of a None string field
    (FORMS); none_num: the slot of a None number (its value is never read)."""
    n = len(schema)
    opt = [c for c, (_, o) in enumerate(schema) if o]
    words = [0] * ((len(opt) + 63) // 64)  # calcBitmapSize: whole 8-byte words
    for k, c in enumerate(opt):
        if values[c] is None:
            words[k >> 6] |= 1 << (k & 63)  # bit k = the k-th Option field is None
    slots, payload = [], b""
    for c, (t, _) in enumerate(schema):
        v = values[c]
        if t != T_STR:
            slots.append(none_num & M64 if v is None else _fixed_slot(t, v))
            continue
        rel = 8 * n + 8 + len(payload) - 8 * c  # (numSerializedElements + 1 - idx) * 8 + varlenSize, FlattenedTuple.cc:801
        text = (null_text + b"\0" if none_str == "payload" else b"") if v is None else v + b"\0"
        slots.append(rel | (len(text) << 32))
        payload += text
    if none_str == "zero_slot" and not payload:
        slots = [0 if t == T_STR else s for s, (t, _) in zip(slots, schema)]
    has_var = any(t == T_STR for t, _ in schema)
    return (struct.pack("<%dQ" % len(words), *words) + struct.pack("<%dQ" % n, *slots)
            + (struct.pack("<q", len(payload)) if has_var else b"") + payload)


def exact_alloc(partition_bytes):
    """A partition holds max(partition_bytes, what the row needs): a row larger than the capacity gets a partition of exactly its
    size, which is what K5 does. The reference's BitmapAllocator rounds up to whole blocks (Executor.cc:260-288), so there the rows
    after a large one may share its partition (DESIGN.md §6)."""
    return lambda need: max(partition_bytes, need)


def to_partitions(rows, schema, partition_bytes, none_str="empty", none_num=0, alloc=None):
    """rowToMemorySink: a row opens a new partition when bytesWritten + size > capacity. none_str may be one form per row. No rows
    give one empty partition (the reference's sink makes none; K5 hands back one, so a caller always has a partition)."""
    alloc = alloc or exact_alloc(partition_bytes)
    parts, cap, written = [], 0, 0
    for i, vals in enumerate(rows):
        r = serialize_row(vals, schema, none_str if isinstance(none_str, str) else none_str[i], none_num)
        if not parts or written + len(r) > cap:
            cap = alloc(len(r) + 8) - 8
            parts.append([])
            written = 0
        parts[-1].append(r)
        written += len(r)
    return [struct.pack("<q", len(p)) + b"".join(p) for p in parts or [[]]]


def exception_partition(records, in_rows, schema):
    """records: (row, rowNo, ecCode, opID); each record carries the original input row in the canonical form."""
    out = struct.pack("<q", len(records))
    for row, row_no, code, op_id in records:
        r = serialize_row(in_rows[row], schema)
        out += struct.pack("<4q", row_no, code, op_id, len(r)) + r
    return out


def read_row(buf, pos, schema):
    """Deserializer: (values, row length) of the row at buf[pos:]."""
    n = len(schema)
    opt = [c for c, (_, o) in enumerate(schema) if o]
    nw = (len(opt) + 63) // 64
    words = struct.unpack_from("<%dQ" % nw, buf, pos)
    none = {c for k, c in enumerate(opt) if (words[k >> 6] >> (k & 63)) & 1}
    base = pos + 8 * nw
    vals = []
    for c, (t, _) in enumerate(schema):
        s = struct.unpack_from("<Q", buf, base + 8 * c)[0]
        if c in none:
            vals.append(None)
        elif t == T_STR:
            size = s >> 32
            a = base + 8 * c + (s & 0xFFFFFFFF)
            vals.append(bytes(buf[a:a + size - 1]) if size else b"")
        elif t == T_F64:
            vals.append(bits_f64(s))
        elif t == T_BOOL:
            vals.append(bool(s))
        else:
            vals.append(s - (1 << 64) if s >> 63 else s)
    length = 8 * nw + 8 * n
    if any(t == T_STR for t, _ in schema):
        length += 8 + struct.unpack_from("<q", buf, base + 8 * n)[0]
    return vals, length


def read_partitions(parts, schema):
    rows = []
    for p in parts:
        pos = 8
        for _ in range(struct.unpack_from("<q", p, 0)[0]):
            v, ln = read_row(p, pos, schema)
            rows.append(tuple(v))
            pos += ln
    return rows


# ---- columns of rows ---------------------------------------------------------------------------------------------------------
def columns_of(rows, schema):
    """Host columns of rows; an Option field's column always has validity words (the bitmap counts it even without a None)."""
    cols = []
    for c, (t, o) in enumerate(schema):
        vals = [r[c] for r in rows]
        present = np.array([v is not None for v in vals], bool)
        valid = pack_valid(present) if o else None
        if t == T_STR:
            enc = [v if v is not None else b"" for v in vals]
            off = np.zeros(len(enc) + 1, np.uint32)
            np.cumsum([len(e) for e in enc], out=off[1:])
            cols.append(Column(T_STR, np.frombuffer(b"".join(enc), np.uint8).copy(), off, valid))
        else:
            bits = np.array([0 if v is None else _fixed_slot(t, v) for v in vals], np.uint64)
            cols.append(Column(t, bits.view(np.float64) if t == T_F64 else bits.view(np.int64), None, valid))
    return cols


def values_of(cols):
    """Rows of host columns: bool columns stay integers, so any slot value other than 0 / 1 would show."""
    n = len(cols[0]) if cols else 0
    out = []
    for col in cols:
        pres = np.ones(n, bool) if col.valid is None else unpack_valid(col.valid, n)
        if col.type == T_STR:
            raw, o = col.data.tobytes(), col.offsets
            vals = [raw[int(o[i]):int(o[i + 1])] for i in range(n)]
        elif col.type == T_F64:
            vals = col.data.tolist()
        else:
            vals = np.asarray(col.data).view(np.int64).tolist()
        out.append([v if p else None for v, p in zip(vals, pres.tolist())])
    return [tuple(r) for r in zip(*out)]


def bit_rows(rows, schema):
    """Rows with every fixed-width value as its slot bits, so that NaN payloads and -0.0 compare exactly."""
    return [tuple(v if v is None or t == T_STR else _fixed_slot(t, v) for v, (t, _) in zip(r, schema)) for r in rows]


def assert_columns(got_cols, got_valid, rows, schema, what=""):
    """The columns a block holds against the rows it was read from: None becomes 0 / "" with a clear present bit."""
    want = columns_of(rows, schema)
    assert len(got_cols) == len(schema)
    for c, (g, gv, w, (t, o)) in enumerate(zip(got_cols, got_valid, want, schema)):
        tag = f"{what} column {c}"
        assert g.type == t, tag
        if o:
            assert gv is not None and np.array_equal(gv, w.valid), f"{tag}: validity words {gv!r} vs {w.valid!r}"
        else:
            assert gv is None, tag
        if t == T_STR:
            assert np.array_equal(g.offsets, w.offsets), f"{tag}: offsets differ from row {np.flatnonzero(g.offsets != w.offsets)[:1]}"
            assert g.data.tobytes() == w.data.tobytes(), f"{tag}: string bytes differ"
        else:
            gb, wb = np.ascontiguousarray(g.data).view(np.uint64), np.ascontiguousarray(w.data).view(np.uint64)
            bad = np.flatnonzero(gb != wb)
            assert bad.size == 0, f"{tag}: bits differ at rows {bad[:8].tolist()}"


# ---- the value matrix --------------------------------------------------------------------------------------------------------
I64_EDGES = [0, 1, -1, I64_MIN, I64_MAX, I64_MIN + 1, (1 << 32) - 1, 1 << 32, -(1 << 32), 1 << 31]
F64_EDGE_BITS = [0x0000000000000000, 0x8000000000000000, 0x7FF8000000000001, 0x7FF0000000000001, 0xFFF8000000000ABC, 0x7FF4000000000000,
                 0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001, 0x3FF8000000000000, 0xFFFFFFFFFFFFFFFF]
STR_EDGES = [b"", b"\0", b"\0\0", b"a\0b", b"\xff", b"\xc3\x28", b"\x80\x00\x80", b"\xed\xa0\x80", b"caf\xc3\xa9", b"N/A", b"x" * 300]


def _value(t, rng, i):
    if t == T_I64:
        return I64_EDGES[i] if i < len(I64_EDGES) else int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64))
    if t == T_F64:
        return bits_f64(F64_EDGE_BITS[i % len(F64_EDGE_BITS)] if i % 3 else int(rng.integers(0, 1 << 63)) * 2 + (i & 1))
    if t == T_BOOL:
        return bool(rng.integers(0, 2))
    if i < len(STR_EDGES):
        return STR_EDGES[i]
    return rng.integers(0, 256, int(rng.integers(0, 301)), dtype=np.uint8).tobytes()  # lengths 0-300, any byte


def _is_none(pattern, i, n, rng):
    return {"none": False, "all": True, "alternating": i % 2 == 1, "random": rng.random() < 0.4}[pattern]


def make_rows(schema, n, pattern, seed):
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        rows.append(tuple(None if o and _is_none(pattern, i, n, rng) else _value(t, rng, i) for t, o in schema))
    return rows


def mixed_forms(n):
    return [FORMS[i % 3] for i in range(n)]


SCHEMAS = {
    "i64": [(T_I64, False)], "opt_i64": [(T_I64, True)], "f64": [(T_F64, False)], "opt_f64": [(T_F64, True)],
    "bool": [(T_BOOL, False)], "opt_bool": [(T_BOOL, True)], "str": [(T_STR, False)], "opt_str": [(T_STR, True)],
    "str_first": [(T_STR, True), (T_I64, False), (T_F64, True), (T_BOOL, False)],
    "str_middle": [(T_I64, True), (T_STR, True), (T_BOOL, True)],
    "str_last": [(T_F64, False), (T_BOOL, True), (T_STR, True)],
    "several_str": [(T_STR, True), (T_I64, False), (T_STR, False), (T_STR, True), (T_F64, True)],
    "no_str": [(T_I64, True), (T_F64, False), (T_BOOL, True)],
    "only_opt_str": [(T_STR, True), (T_STR, True), (T_STR, True)],
    "cols_63": [((T_I64, T_F64, T_BOOL, T_STR)[c % 4], c % 3 != 1) for c in range(63)],
    "cols_64": [((T_STR, T_I64, T_F64, T_BOOL)[c % 4], True) for c in range(64)],
}
PATTERNS = ["none", "all", "alternating", "random"]


def matrix():
    """(name, schema, rows, per-row None-string forms) of every schema and None pattern."""
    out = []
    for k, (name, schema) in enumerate(SCHEMAS.items()):
        n = 120 if len(schema) > 8 else 300
        for j, pattern in enumerate(PATTERNS):
            rows = make_rows(schema, n, pattern, 100 * k + j)
            out.append((f"{name}-{pattern}", schema, rows, mixed_forms(n)))
    return out


# ---- a large block built with numpy -------------------------------------------------------------------------------------------
BIG_SCHEMA = [(T_I64, False), (T_STR, True)]


def big_partitions(n, rows_per_part, seed):
    """Partitions of (a: i64, s: Option[str]) rows, built with numpy; row i's string has (7 i) % 13 bytes, every fifth row is None,
    half of them in the payload form ("N/A\\0"). Returns (partitions, a, string lengths, None mask, expected string bytes)."""
    rng = np.random.default_rng(seed)
    idx = np.arange(n, dtype=np.int64)
    a = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64)
    L = (idx * 7) % 13
    none = idx % 5 == 3
    pay = none & (idx % 10 == 3)
    plen = np.where(none, np.where(pay, 4, 0), L + 1)
    parts, keep_bytes = [], []
    for lo in range(0, max(n, 1), rows_per_part):
        hi = min(n, lo + rows_per_part)
        m = hi - lo
        pl = plen[lo:hi]
        size = 32 + pl
        start = np.zeros(m, np.int64)
        np.cumsum(size[:-1], out=start[1:]) if m else None
        buf = np.zeros(8 + int(size.sum()), np.uint8)
        buf[:8] = np.frombuffer(struct.pack("<q", m), np.uint8)
        fixed = np.zeros((m, 4), np.uint64)
        fixed[:, 0] = none[lo:hi].astype(np.uint64)                                        # bitmap word
        fixed[:, 1] = a[lo:hi].view(np.uint64)
        fixed[:, 2] = np.uint64(16) | (pl.astype(np.uint64) << np.uint64(32))             # s: bytes at slot + 16 (after the total)
        fixed[:, 3] = pl.astype(np.uint64)                                                 # var-len total
        fb = fixed.view(np.uint8).reshape(m, 32)
        buf[(8 + start)[:, None] + np.arange(32)] = fb
        tot = int(pl.sum())
        rid = np.repeat(np.arange(m), pl)
        within = np.arange(tot) - np.repeat(np.cumsum(pl) - pl, pl)
        text = rng.integers(1, 256, tot, dtype=np.uint8)
        text[within == pl[rid] - 1] = 0                                                    # the NUL of every string
        na = pay[lo:hi][rid] & (within < 3)
        text[na] = np.frombuffer(b"N/A", np.uint8)[within[na]]
        buf[np.repeat(8 + start + 32, pl) + within] = text
        parts.append(buf.tobytes())
        keep_bytes.append(text[~none[lo:hi][rid] & (within < pl[rid] - 1)])
    return parts, a, np.where(none, 0, L), none, np.concatenate(keep_bytes) if keep_bytes else np.zeros(0, np.uint8)


# =============================================================================================================================
# CPU part
# =============================================================================================================================
def test_restatement_reproduces_the_hand_derived_option_row():
    """The row of test_option.py::test_oracle_row_bytes_with_option_fields_hand_derived."""
    schema = [(T_I64, True), (T_STR, False), (T_STR, True), (T_STR, True), (T_I64, False)]
    row = struct.pack("<q", 0b011) + struct.pack("<5q", 0, 40 | (3 << 32), 35, 27 | (2 << 32), 7) + struct.pack("<q", 5) + b"ab\0x\0"
    assert serialize_row((None, b"ab", None, b"x", 7), schema) == row
    assert to_partitions([(None, b"ab", None, b"x", 7)], schema, 1 << 20) == [struct.pack("<q", 1) + row]
    assert read_partitions([struct.pack("<q", 1) + row], schema) == [(None, b"ab", None, b"x", 7)]


def test_hand_derived_rows_whose_only_strings_are_none():
    """(k: i64 = 5, s: Option[str] = None, t: Option[str] = None) in each form."""
    schema = [(T_I64, False), (T_STR, True), (T_STR, True)]
    vals = (5, None, None)
    head = struct.pack("<q", 0b11) + struct.pack("<q", 5)
    # "empty": offsets still point where the payload starts (FlattenedTuple.cc:801: (3 + 1 - 1) * 8 + 0, (3 + 1 - 2) * 8 + 0)
    assert serialize_row(vals, schema, "empty") == head + struct.pack("<2q", 24, 16) + struct.pack("<q", 0)
    # "zero_slot": no var-len bytes in the row, so Serializer.cc:1071 never fills the slots
    assert serialize_row(vals, schema, "zero_slot") == head + struct.pack("<2q", 0, 0) + struct.pack("<q", 0)
    # "payload": both cells were "N/A": slot s at 24 with size 4, slot t at 16 + 4 with size 4, total 8
    assert serialize_row(vals, schema, "payload") == head + struct.pack("<2q", 24 | (4 << 32), 20 | (4 << 32)) + struct.pack("<q", 8) + b"N/A\0N/A\0"
    for f in FORMS:
        assert read_partitions(to_partitions([vals], schema, 4096, f), schema) == [vals]


def test_hand_derived_row_with_a_none_na_cell_before_a_string():
    """(s: Option[str] = None read from "N/A", u: str = "xy"): FlattenedTuple::serialize copies the cell's text for the None field
    and the next field's bytes follow it."""
    schema = [(T_STR, True), (T_STR, False)]
    row = struct.pack("<q", 1) + struct.pack("<2q", 24 | (4 << 32), 20 | (3 << 32)) + struct.pack("<q", 7) + b"N/A\0xy\0"
    assert serialize_row((None, b"xy"), schema, "payload") == row
    # the same row in the canonical form has no bytes for s and u's bytes move up
    assert serialize_row((None, b"xy"), schema, "empty") == struct.pack("<q", 1) + struct.pack("<2q", 24, 16 | (3 << 32)) + struct.pack("<q", 3) + b"xy\0"
    assert read_partitions([struct.pack("<q", 1) + row], schema) == [(None, b"xy")]


def test_hand_derived_row_with_64_option_fields():
    """64 Option[i64] fields (TPLX_MAX_COLS): one bitmap word, field 63 is its top bit."""
    schema = [(T_I64, True)] * 64
    vals = tuple(None if c in (0, 62, 63) else c for c in range(64))
    want = struct.pack("<Q", (1 << 0) | (1 << 62) | (1 << 63)) + struct.pack("<64q", *[0 if v is None else v for v in vals])
    assert serialize_row(vals, schema) == want
    assert serialize_row(vals, schema, none_num=-1)[8:16] == b"\xff" * 8
    assert read_partitions(to_partitions([vals], schema, 1024), schema) == [vals]


def _ocols(rows, schema):
    return columns_of(rows, schema)


def test_oracle_agrees_with_the_restatement_over_the_matrix(built):
    """The C oracle (a second subject, like K5) writes the canonical form byte for byte: partitions at three sizes and the exception
    partition of every third row."""
    for name, schema, rows, _ in matrix():
        cols = _ocols(rows, schema)
        for pb in (256, 4096, 1 << 20):
            if any(len(serialize_row(r, schema)) + 8 > pb for r in rows):
                continue  # the oracle has no notion of an allocator; rows larger than a partition are K5's own case
            assert po.to_partitions(cols, len(rows), pb) == to_partitions(rows, schema, pb), (name, pb)
        recs = [(i, 1000 + 2 * i, 3 + i % 5, 100001 + i % 2) for i in range(0, len(rows), 3)]
        exc = np.array([(r, no, code, op) for r, no, code, op in recs], dtype=[("row", "<i8"), ("row_no", "<i8"), ("code", "<i8"), ("op_id", "<i8")])
        assert po.exception_partition(cols, exc) == exception_partition(recs, rows, schema), name
    assert po.to_partitions(_ocols([], SCHEMAS["str_first"]), 0, 4096) == to_partitions([], SCHEMAS["str_first"], 4096) == [bytes(8)]


def test_reader_reads_every_form_back():
    for name, schema, rows, forms in matrix():
        for f in list(FORMS) + [forms]:
            got = read_partitions(to_partitions(rows, schema, 4096, f, none_num=0x5A5A5A5A5A5A5A5A), schema)
            assert bit_rows(got, schema) == bit_rows(rows, schema), name


def test_matrix_reaches_its_edges():
    """Row starts at every offset mod 16 (unaligned slots) in every narrow string schema that has string bytes."""
    for name, schema, rows, forms in matrix():
        if not any(t == T_STR for t, _ in schema) or name.endswith("-all") or len(schema) > 8:
            continue
        (p,) = to_partitions(rows, schema, 1 << 30, forms)
        starts, pos = set(), 8
        for r, f in zip(rows, forms):
            starts.add(pos % 16)
            pos += len(serialize_row(r, schema, f))
        assert starts == set(range(16)), name
    assert any(len(r[0]) == 300 for r in make_rows(SCHEMAS["str"], 300, "none", 0))


def test_numpy_partitions_match_the_restatement():
    parts, a, L, none, kept = big_partitions(3000, 1024, 1)
    forms = ["payload" if (i % 5 == 3 and i % 10 == 3) else "empty" for i in range(3000)]
    rows = read_partitions(parts, BIG_SCHEMA)
    assert [r[0] for r in rows] == a.tolist()
    assert [r[1] is None for r in rows] == none.tolist()
    want = to_partitions(rows, BIG_SCHEMA, 1 << 30, forms)[0][8:]
    assert b"".join(p[8:] for p in parts) == want
    assert kept.tobytes() == b"".join(r[1] for r in rows if r[1] is not None)


def test_reference_allocator_departure():
    """A row larger than the capacity: K5 closes its partition behind it; the reference's block allocator may leave room after it."""
    schema = [(T_STR, False)]
    rows = [(b"a",), (b"x" * 83,), (b"b",)]  # rows of 18, 100 and 18 bytes; capacity 56
    assert [len(p) for p in to_partitions(rows, schema, 64)] == [8 + 18, 8 + 100, 8 + 18]
    blocks = to_partitions(rows, schema, 64, alloc=lambda need: -(-need // 64) * 64)
    assert [struct.unpack_from("<q", p)[0] for p in blocks] == [1, 2]  # the large row's two blocks have room for the next one


# =============================================================================================================================
# GPU part
# =============================================================================================================================
def passthrough(schema, option=False):
    """A stage that hands its input columns out unchanged. option=False declares every field plain, so a block with Option fields is
    read as stored (placeholders included) and its validity comes from Block.validity; option=True carries the validity through."""
    names = ["c%d" % c for c in range(len(schema))]
    sc = frontend.StageCompiler([t for t, _ in schema], names, [c for c, (_, o) in enumerate(schema) if o] if option else [])
    return sc.finish_memory()


def block_of(parts, schema):
    return backend.Block.from_partitions(0, parts, [t for t, _ in schema], [c for c, (_, o) in enumerate(schema) if o])


def read_block(parts, schema):
    blk = block_of(parts, schema)
    st = backend.Stage(passthrough(schema))
    try:
        res = st.run(blk)
        cols = res.columns() if blk.n_rows else [None] * len(schema)
        valid = [blk.validity(c) for c in range(len(schema))]
        n = blk.n_rows
        res.free()
    finally:
        st.close()
        blk.free()
    return n, cols, valid


def check_read(parts, schema, rows, what=""):
    n, cols, valid = read_block(parts, schema)
    assert n == len(rows), what
    if n:
        assert_columns(cols, valid, rows, schema, what)
    return cols


def _ids(cases):
    return [c[0] for c in cases]


MATRIX = matrix()


@pytest.mark.gpu
@pytest.mark.parametrize("case", MATRIX, ids=_ids(MATRIX))
def test_gpu_block_from_partitions_matrix(gpu, case):
    """Every schema and None pattern, the three None-string forms mixed row by row, several partitions."""
    name, schema, rows, forms = case
    for f in (forms, "payload"):
        parts = to_partitions(rows, schema, 2048, f, none_num=0x5A5A5A5A5A5A5A5A)
        check_read(parts, schema, rows, name)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 999, 1000, 2049])
def test_gpu_payload_nones_at_the_end_and_before_long_strings(gpu, n):
    """Payload-form None cells as the last rows with bytes, and right before rows with long strings: their text must not reach
    any other row's bytes, and the column holds no byte of it."""
    schema = [(T_I64, False), (T_STR, True), (T_STR, False)]
    rng = np.random.default_rng(n)
    rows = []
    for i in range(n):
        s = None if (i % 7 == 0 or i >= n - 3) else rng.integers(0, 256, 8 + i % 300, dtype=np.uint8).tobytes()
        rows.append((i, s, b"" if i >= n - 3 else b"long" * (2 + i % 40)))
    for ps in (64 << 10, 1 << 30):
        check_read(to_partitions(rows, schema, ps, "payload"), schema, rows, f"n={n}")
    # the layout of the first report: a None "N/A" cell in row 0, every later row with a string of 8 bytes or more
    rows = [(0, None, b"")] + [(i, b"s%07d" % i, b"") for i in range(1, 1000)]
    check_read(to_partitions(rows, schema, 1 << 20, "payload"), schema, rows, "row 0")


@pytest.mark.gpu
def test_gpu_string_of_one_mib(gpu):
    schema = [(T_STR, True), (T_I64, False), (T_STR, False)]
    big = bytes(range(256)) * 4096 + b"\0\xff"
    rows = [(b"a", 1, b"b"), (big, 2, big[::-1]), (None, 3, b""), (b"", 4, big[:7])]
    check_read(to_partitions(rows, schema, 1 << 20, "payload"), schema, rows)


@pytest.mark.gpu
def test_gpu_empty_partitions_slack_and_one_row_partitions(gpu):
    schema = SCHEMAS["several_str"]
    rows = make_rows(schema, 200, "random", 7)
    parts = to_partitions(rows, schema, 1024, mixed_forms(200))
    empty = struct.pack("<q", 0)
    check_read([empty] + parts[:2] + [empty, empty] + parts[2:] + [empty], schema, rows, "empty partitions")
    check_read([p + b"\xee" * (1 + k % 17) for k, p in enumerate(parts)], schema, rows, "slack bytes")
    check_read([], schema, [], "no partitions")
    check_read([empty], schema, [], "one empty partition")
    many = make_rows(schema, 3000, "alternating", 8)
    forms = mixed_forms(3000)
    one_each = [struct.pack("<q", 1) + serialize_row(r, schema, f) for r, f in zip(many, forms)]
    check_read(one_each, schema, many, "one row per partition")


@pytest.mark.gpu
def test_gpu_malformed_partitions_are_refused(gpu):
    schema = [(T_I64, False), (T_STR, True)]
    good = to_partitions([(1, b"abc"), (2, None)], schema, 4096)[0]
    row0 = serialize_row((1, b"abc"), schema)
    bad = {
        "negative numRows": struct.pack("<q", -1) + good[8:],
        "numRows past the end": struct.pack("<q", 3) + good[8:],
        "truncated row": good[:-1],
        "truncated fixed part": good[:8 + 20],
        # row = bitmap, 2 slots, var-len total at byte 24, payload "abc\0"
        "var-len total past the end": struct.pack("<q", 1) + row0[:24] + struct.pack("<q", 5) + row0[32:],
        "var-len total near 2^64": struct.pack("<q", 1) + row0[:24] + struct.pack("<Q", M64) + row0[32:],
        "var-len total of 2^63": struct.pack("<q", 1) + row0[:24] + struct.pack("<Q", 1 << 63) + row0[32:],
        "shorter than a header": b"\0" * 7,
    }
    assert struct.unpack_from("<q", row0, 24)[0] == 4 and len(row0) == 36
    for what, p in bad.items():
        try:
            block_of([good, p], schema).free()
        except backend.GpuBackendError as e:
            assert re.search(r"failed \(-4\).*malformed", str(e)), (what, str(e))
        else:
            pytest.fail(f"{what}: accepted")
    check_read([good], schema, [(1, b"abc"), (2, None)])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049])
def test_gpu_row_counts(gpu, n):
    schema = SCHEMAS["several_str"]
    rows = make_rows(schema, n, "random", 1000 + n)
    check_read(to_partitions(rows, schema, 8192, mixed_forms(n)), schema, rows, f"n={n}")


@pytest.mark.gpu
def test_gpu_block_over_1024_scan_blocks(gpu):
    """2^21 + 2049 rows: the string-length scan has 1,026 block sums, so scan_of_sums takes its second round."""
    n = (1 << 21) + 2049
    parts, a, L, none, kept = big_partitions(n, 1 << 16, 2)
    _, cols, valid = read_block(parts, BIG_SCHEMA)
    assert np.array_equal(cols[0].data.view(np.int64), a)
    assert valid[0] is None and np.array_equal(valid[1], pack_valid(~none))
    off = np.zeros(n + 1, np.int64)
    np.cumsum(L, out=off[1:])
    assert np.array_equal(cols[1].offsets.astype(np.int64), off)
    assert np.array_equal(cols[1].data, kept)


# ---- the output direction ----------------------------------------------------------------------------------------------------
def result_schema(cols):
    return [(c.type, c.valid is not None) for c in cols]


def check_result_partitions(res, sizes=(64, 4096, 1 << 20), what=""):
    """K5's partitions of a result against the restatement's serialization of the result's own columns."""
    cols = res.columns()
    schema = result_schema(cols)
    rows = values_of(cols)
    for pb in sizes:
        assert res.partitions(pb) == to_partitions(rows, schema, pb), (what, pb)
    return rows


def _option_input(n, seed):
    schema = [(T_I64, True), (T_STR, False), (T_STR, True), (T_F64, True), (T_BOOL, True)]
    rows = make_rows(schema, n, "random", seed)
    return schema, rows


@pytest.mark.gpu
def test_gpu_result_partitions_of_a_memory_stage_with_option_outputs(gpu):
    schema, rows = _option_input(3000, 11)
    parts = to_partitions(rows, schema, 8192, mixed_forms(len(rows)))
    blk = block_of(parts, schema)
    st = backend.Stage(passthrough(schema, option=True))
    res = st.run(blk)
    try:
        assert bit_rows(check_result_partitions(res, what="pass-through"), schema) == bit_rows(rows, schema)
        # the round trip: whatever form the input had, the output is the canonical form of the input's values
        for pb in (8192, 1 << 20):
            assert res.partitions(pb) == to_partitions(rows, schema, pb)
    finally:
        res.free()
        st.close()
        blk.free()


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_gpu_round_trip_comes_back_canonical(gpu, form):
    for name in ("str_first", "several_str", "only_opt_str", "no_str", "opt_str"):
        schema = SCHEMAS[name]
        rows = make_rows(schema, 500, "alternating", 5)
        blk = block_of(to_partitions(rows, schema, 4096, form, none_num=-1), schema)
        st = backend.Stage(passthrough(schema, option=True))
        res = st.run(blk)
        try:
            for pb in (4096, 1 << 20):
                assert res.partitions(pb) == to_partitions(rows, schema, pb), (name, form)
        finally:
            res.free()
            st.close()
            blk.free()


@pytest.mark.gpu
def test_gpu_result_partitions_of_an_aggregate(gpu):
    """The agg_out branch: one row with one slot per accumulator, whatever the partition size (LocalBackend.cc:1180-1207)."""
    n = 5000
    rng = np.random.default_rng(12)
    cols = [Column(T_I64, rng.integers(-1000, 1000, n)), Column(T_F64, rng.standard_normal(n))]
    sc = frontend.StageCompiler([T_I64, T_F64], ["v", "f"])
    prog = sc.finish_aggregate(lambda a, x: (a[0] + x["v"], min(a[1], x["f"]), a[2] + 1), lambda a, b: (a[0] + b[0], min(a[1], b[1]), a[2] + b[2]),
                               (0, 1e300, 0), 100001)
    st = backend.Stage(prog)
    res = st.run(backend.Block.upload(0, cols, n))
    try:
        bits = res.aggregate_bits()
        schema = [(T_I64, False)] * len(bits)
        assert bits[0] == int(cols[0].data.sum()) & M64 and bits[2] == n
        for pb in (9, 64, 1 << 20):
            assert res.partitions(pb) == to_partitions([tuple(bits)], schema, 1 << 20)
    finally:
        res.free()
        st.close()


@pytest.mark.gpu
def test_gpu_result_partitions_of_aggregate_by_key_with_option_keys(gpu):
    rng = np.random.default_rng(13)
    n = 4000
    k0 = [None if rng.random() < 0.2 else int(v) for v in rng.integers(-3, 4, n)]
    s = [None if rng.random() < 0.3 else ["", "a", "\xe4", "日本語"][int(rng.integers(0, 4))] for _ in range(n)]
    v = rng.integers(-100, 100, n).tolist()
    cols = [Column.from_values(k0, T_I64), Column.from_values(s, T_STR), Column.from_values(v, T_I64)]
    sc = frontend.StageCompiler([T_I64, T_STR, T_I64], ["k0", "s", "v"], option_cols=[0, 1])
    st = backend.Stage(sc.finish_hash(["k0", "s"], lambda a, x: a + x["v"], lambda a, b: a + b, 0, 100001))
    st.run(backend.Block.upload(0, cols, n)).info
    res = st.hash_finish(0)
    try:
        got = check_result_partitions(res, what="aggregateByKey")
        want = {}
        for a, b, c in zip(k0, s, v):
            key = (a, None if b is None else b.encode())
            want[key] = want.get(key, 0) + c
        assert sorted(got, key=repr) == sorted([k + (x,) for k, x in want.items()], key=repr)
        assert any(r[0] is None for r in got) and any(r[1] is None for r in got)
    finally:
        res.free()
        st.close()


@pytest.mark.gpu
def test_gpu_result_partitions_of_a_left_outer_join(gpu):
    rng = np.random.default_rng(14)
    left = [Column.from_values(rng.integers(0, 60, 700).tolist(), T_I64), Column.from_values(["l%d" % i * (i % 4) for i in range(700)], T_STR)]
    right = [Column.from_values(list(range(0, 80, 2)), T_I64), Column.from_values(["r\xff%d" % i for i in range(40)], T_STR),
             Column.from_values([None if i % 3 == 0 else float(i) for i in range(40)], T_F64)]
    lb, rb = backend.Block.upload(0, left, 700), backend.Block.upload(0, right, 40)
    jn = backend.Join(rb, [T_I64, T_STR, T_F64], 0)
    jr = jn.probe(lb, [T_I64, T_STR], 0, left_outer=True)
    try:
        rows = check_result_partitions(jr, what="left join")
        assert len(rows) == 700 and any(r[2] is None for r in rows) and any(r[3] is None and r[2] is not None for r in rows)
    finally:
        jr.free()
        jn.free()
        lb.free()
        rb.free()


@pytest.mark.gpu
def test_gpu_result_partitions_of_merged_resolved_rows(gpu):
    n = 3000
    rng = np.random.default_rng(15)
    k = rng.integers(0, 7, n)
    cols = [Column.from_values(k.tolist(), T_I64), Column.from_values(["w%d" % (v % 11) * int(v % 3) for v in range(n)], T_STR)]
    sc = frontend.StageCompiler([T_I64, T_STR], ["k", "s"])
    sc.add_map(lambda x: (100 // x["k"], x["s"].upper() + "!", x["k"]), 100001)
    st = backend.Stage(sc.finish_memory())
    res = st.run_host(0, cols, n)
    exc = res.exceptions()
    rr = [(int(e["row_no"]), -1, "resolved-%d" % int(e["row"]), int(e["row"])) for j, e in enumerate(exc) if j % 3 != 2]
    blk = backend.Block.upload(0, [Column.from_values([r[1] for r in rr], T_I64), Column.from_values([r[2] for r in rr], T_STR),
                                   Column.from_values([r[3] for r in rr], T_I64)], len(rr))
    merged = res.merge_resolved(blk, [r[0] for r in rr])
    try:
        rows = check_result_partitions(merged, what="merge_resolved")
        assert len(rows) == n - (len(exc) - len(rr))
    finally:
        merged.free()
        res.free()
        st.close()


# ---- the split -----------------------------------------------------------------------------------------------------------------
def _str_result(strs):
    """A result of (i: i64, s: Option[str]) rows from a pass-through stage; a row is 32 + len(s) + 1 bytes (32 for None)."""
    schema = [(T_I64, False), (T_STR, True)]
    rows = [(i, s) for i, s in enumerate(strs)]
    blk = block_of(to_partitions(rows, schema, 1 << 30), schema)
    st = backend.Stage(passthrough(schema, option=True))
    res = st.run(blk)
    return res, (st, blk), rows, schema


def _free(res, keep):
    res.free()
    keep[0].close()
    keep[1].free()


def _split(parts):
    return [struct.unpack_from("<q", p)[0] for p in parts]


@pytest.mark.gpu
def test_gpu_split_at_capacity(gpu):
    strs = [b"x" * 7] * 6 + [None, b"", b"x" * 200, b"yy", None]  # 40 B rows, then 32, 33, 233, 35, 32
    res, keep, rows, schema = _str_result(strs)
    try:
        for pb in [8 + 40, 8 + 39, 8 + 41, 8 + 80, 8 + 79, 8 + 120, 8 + 72, 8 + 233, 8 + 232, 9, 10, 1 << 20]:
            assert res.partitions(pb) == to_partitions(rows, schema, pb), pb
        assert _split(res.partitions(8 + 40)) == [1] * 6 + [1, 1, 1, 1, 1]            # a row exactly at capacity
        assert _split(res.partitions(8 + 39)) == [1] * 11                             # one byte over: a partition of its own
        assert _split(res.partitions(8 + 120)) == [3, 3, 2, 1, 2]                     # 3 x 40 = capacity; the 233 B row alone
        assert _split(res.partitions(8 + 72)) == [1, 1, 1, 1, 1, 2, 1, 1, 2]          # 40 + 32 = capacity
        assert _split(res.partitions(9)) == [1] * 11
        with pytest.raises(backend.GpuBackendError, match=r"failed \(-4\)"):
            res.partitions(8)
    finally:
        _free(res, keep)


@pytest.mark.gpu
def test_gpu_split_of_a_row_larger_than_the_capacity(gpu):
    strs = [b"a", b"b", b"x" * 5000, b"c", None, b"x" * 6000, b"x" * 6000]
    res, keep, rows, schema = _str_result(strs)
    try:
        parts = res.partitions(4096)
        assert parts == to_partitions(rows, schema, 4096)
        assert _split(parts) == [2, 1, 2, 1, 1]
    finally:
        _free(res, keep)


@pytest.mark.gpu
def test_gpu_split_of_no_rows(gpu):
    res, keep, rows, schema = _str_result([])
    try:
        assert res.partitions(64) == [bytes(8)] == to_partitions([], schema, 64)
    finally:
        _free(res, keep)


def _raw_partitions(res, pb, max_parts):
    need, nparts = ct.c_uint64(), ct.c_uint32()
    rc = backend.lib().tplx_gpu_result_partitions(res._h, pb, None, 0, ct.byref(need), None, 0, ct.byref(nparts))
    if rc:
        return rc, 0
    buf = np.empty(max(need.value, 8), np.uint8)
    offs = (ct.c_uint64 * (max_parts + 1))()
    return backend.lib().tplx_gpu_result_partitions(res._h, pb, buf.ctypes.data, buf.nbytes, ct.byref(need), offs, max_parts,
                                                    ct.byref(nparts)), nparts.value


@pytest.mark.gpu
def test_gpu_split_partition_count_limits(gpu):
    """65,536 partitions are accepted, 65,537 give TPLX_E_OVERFLOW; max_parts below the count needed gives TPLX_E_BADARG."""
    schema = [(T_I64, False)]
    for n, rc_want in ((1 << 16, 0), ((1 << 16) + 1, E_OVERFLOW)):
        vals = np.arange(n, dtype=np.int64) * -7
        st = backend.Stage(passthrough(schema))
        res = st.run(backend.Block.upload(0, [Column(T_I64, vals)], n))
        try:
            if rc_want:
                with pytest.raises(backend.GpuBackendError, match=r"failed \(-7\)"):
                    res.partitions(16)
                continue
            t0 = time.perf_counter()
            parts = res.partitions(16)
            ms = (time.perf_counter() - t0) * 1e3
            print(f"\n65,536 one-row partitions: Result.partitions took {ms:.1f} ms (H100; cols_to_rows' linear partition search)")
            assert parts == to_partitions([(int(v),) for v in vals], schema, 16)
            assert _raw_partitions(res, 16, (1 << 16) - 1) == (E_BADARG, 1 << 16)
            assert _raw_partitions(res, 16, 1 << 16) == (0, 1 << 16)
        finally:
            res.free()
            st.close()


# ---- exception partitions -------------------------------------------------------------------------------------------------------
def _records(res):
    e = res.exceptions()
    return [(int(r["row"]), int(r["row_no"]), int(r["code"]), int(r["op_id"])) for r in e]


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_gpu_exception_partition_of_option_inputs(gpu, form):
    """A stage over Option inputs (its block gets `is None` companions, which the exception rows leave out): a None in `a` raises
    TypeError, and the exception partition carries the canonical form of the original rows, whatever form they were read in."""
    schema, rows = _option_input(2500, 16)
    blk = block_of(to_partitions(rows, schema, 16384, form, none_num=-1), schema)
    names = ["a", "s", "t", "f", "b"]
    sc = frontend.StageCompiler([t for t, _ in schema], names, [0, 2, 3, 4])
    sc.add_map(lambda x: (x["a"] + 1, x["s"], x["t"]), 100001)
    st = backend.Stage(sc.finish_memory())
    res = st.run(blk)
    try:
        recs = _records(res)
        assert [r[0] for r in recs] == [i for i, r in enumerate(rows) if r[0] is None] and recs
        assert res.exception_partition() == exception_partition([(r, no, code, op) for r, no, code, op in recs], rows, schema)
    finally:
        res.free()
        st.close()
        blk.free()


@pytest.mark.gpu
def test_gpu_exception_partition_after_a_prefilter(gpu):
    schema = [(T_I64, False), (T_STR, False), (T_I64, False)]
    rng = np.random.default_rng(17)
    n = 6000
    rows = [(int(rng.integers(-5, 5)), b"t%dx\xff" % i * (i % 5), int(rng.integers(0, 4))) for i in range(n)]
    sc = frontend.StageCompiler([T_I64, T_STR, T_I64], ["k", "s", "d"])
    sc.add_filter(lambda x: x["k"] > 0, 100001)
    sc.add_map(lambda x: (x["s"].replace("t", "T").replace("x", "yy") + str(x["k"]), 100 // x["d"]), 100002)
    prog = sc.finish_memory()
    assert prog.prefilter is not None
    st = backend.Stage(prog)
    blk = block_of(to_partitions(rows, schema, 1 << 16), schema)
    res = st.run(blk)
    try:
        recs = _records(res)
        assert [r[0] for r in recs] == [i for i, r in enumerate(rows) if r[0] > 0 and r[2] == 0] and recs
        assert res.exception_partition() == exception_partition(recs, rows, schema)
    finally:
        res.free()
        st.close()
        blk.free()


@pytest.mark.gpu
def test_gpu_exception_partition_of_a_fixed_width_stage(gpu):
    schema = [(T_I64, False), (T_F64, False), (T_BOOL, False)]
    rows = make_rows(schema, 3000, "none", 18)
    rows = [(r[0] % 9 - 4, r[1], r[2]) for r in rows]
    sc = frontend.StageCompiler([t for t, _ in schema], ["a", "f", "b"])
    sc.add_map(lambda x: (100 // x["a"], x["f"] * 2.0), 100001)
    st = backend.Stage(sc.finish_memory())
    assert st.vec_plan() is not None  # the fixed-width row kernel (K1v) runs it
    blk = block_of(to_partitions(rows, schema, 4096), schema)
    res = st.run(blk)
    try:
        recs = _records(res)
        assert [r[0] for r in recs] == [i for i, r in enumerate(rows) if r[0] == 0] and recs
        assert res.exception_partition() == exception_partition(recs, rows, schema)
    finally:
        res.free()
        st.close()
        blk.free()
