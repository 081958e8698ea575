"""Option[T] columns of the CSV source on the CPU: the reference for the device parse, csvops.cuh built for the host against
it, type inference (CSVStatistic with disableNullColumns), type hints, projection of Option columns with their companions and
the typed decode of rows that take the interpreter path.

The reference (`option_reference`) restates decodeCells (codegen/src/FlattenedTuple.cc:1259-1300) over the C oracle's row
splitting and dequoting (oracle/csv_oracle.c, every column read as str without null values) and its scalar decoders: a cell
equal to a null value is None in an Option column, a NULLERROR row in any other column; a non-null cell decodes as in a T column.
"""
import ctypes as ct
import gzip
import os
import random
import subprocess
import typing

import numpy as np
import pytest

from tuplex_b200 import csvsource as cs
from tuplex_b200 import ir
from tuplex_b200.dataset import _compile_stage
from tuplex_b200.pyexec import Op
from oracle import pyoracle as po
from csv_helpers import HERE, T_BOOL, T_F64, T_I64, T_SKIP, T_STR, gen_csv

OPT = ir.C["TPLX_T_OPTION"]
NULLERROR, BADPARSE = 50, 70
NULLS_311 = ["Unspecified", "NO CLUE", "NA", "N/A", "0", ""]


def golden(name: str) -> bytes:
    with gzip.open(os.path.join(HERE, "golden", name + ".gz"), "rb") as f:
        return f.read()


class OptParsed:
    """n_rows, columns (arrays or (bytes, offsets)), valid (per column: validity words or None), rowmap, bad [(row, code)]"""

    def __init__(self, n_rows, columns, valid, rowmap, bad):
        self.n_rows, self.columns, self.valid, self.rowmap, self.bad = n_rows, columns, valid, rowmap, bad


def _words(present):
    n = len(present)
    w = np.zeros((n + 31) // 32, dtype=np.uint32)
    for r, p in enumerate(present):
        if p:
            w[r >> 5] |= np.uint32(1 << (r & 31))
    return w


def option_reference(data: bytes, col_types, header=False, null_values=("",), delimiter=",", quotechar='"') -> OptParsed:
    sel = [c for c, t in enumerate(col_types) if t != T_SKIP]
    base = po.csv_parse(data, [T_STR if t != T_SKIP else T_SKIP for t in col_types], delimiter, quotechar, header, [])
    bad = [(r, code) for r, code, _, _ in base.bad]
    cells = []  # per parsed row: dequoted cells of the selected columns
    for k in range(len(base.rowmap)):
        cells.append([base.columns[j][0][base.columns[j][1][k]:base.columns[j][1][k + 1]] for j in range(len(sel))])
    vals = [[] for _ in sel]
    present = [[] for _ in sel]
    rowmap = []
    kind = {T_I64: "i64", T_F64: "f64", T_BOOL: "bool"}
    for k, row in enumerate(base.rowmap):
        out, code = [], 0
        for j, c in enumerate(sel):
            t, s = col_types[c] & ~OPT, cells[k][j].decode("latin1")
            if s in null_values:
                if not col_types[c] & OPT:
                    code = NULLERROR
                    break
                out.append(None)
                continue
            v = s.encode("latin1") if t == T_STR else po.csv_scalar(kind[t], s)
            if v is None:
                code = BADPARSE
                break
            out.append(v)
        if code:
            bad.append((int(row), code))
            continue
        rowmap.append(int(row))
        for j, v in enumerate(out):
            vals[j].append(v)
            present[j].append(v is not None)
    bad.sort()
    cols, valid = [], []
    for j, c in enumerate(sel):
        t = col_types[c] & ~OPT
        if t == T_STR:
            bs = [v or b"" for v in vals[j]]
            cols.append((b"".join(bs), np.concatenate([[0], np.cumsum([len(b) for b in bs])]).astype(np.uint32)))
        elif t == T_F64:
            cols.append(np.array([0.0 if v is None else v for v in vals[j]], dtype=np.float64))
        else:
            cols.append(np.array([0 if v is None else int(v) for v in vals[j]], dtype=np.int64))
        valid.append(_words(present[j]) if col_types[c] & OPT else None)
    return OptParsed(base.n_rows, cols, valid, np.array(rowmap, dtype=np.uint32), bad)


_SO = None


def _shim():
    global _SO
    if _SO is None:
        so = os.path.join("/tmp", f"csv_option_host_{os.getpid()}.so")
        subprocess.check_call(["g++", "-O1", "-x", "c++", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so,
                               os.path.join(HERE, "csv_option_host.cpp")])
        L = ct.CDLL(so)
        L.hopt_parse.restype = ct.c_void_p
        L.hopt_parse.argtypes = [ct.c_char_p, ct.c_uint32, ct.c_uint8, ct.c_uint8, ct.c_int, ct.c_uint32, ct.c_char_p, ct.c_uint32,
                                 ct.POINTER(ct.c_char_p)]
        for f, rt in (("hopt_fixed", ct.POINTER(ct.c_uint64)), ("hopt_offsets", ct.POINTER(ct.c_uint32)),
                      ("hopt_bytes", ct.POINTER(ct.c_uint8)), ("hopt_valid", ct.POINTER(ct.c_uint32)),
                      ("hopt_rowmap", ct.POINTER(ct.c_uint32)), ("hopt_bad", ct.POINTER(ct.c_uint32))):
            getattr(L, f).restype = rt
        for f in ("hopt_counts", "hopt_type", "hopt_fixed", "hopt_offsets", "hopt_rowmap", "hopt_bad", "hopt_free"):
            getattr(L, f).argtypes = [ct.c_void_p] + ([ct.c_uint32] if f in ("hopt_type", "hopt_fixed", "hopt_offsets") else []) + \
                                     ([ct.POINTER(ct.c_uint32)] if f == "hopt_counts" else [])
        L.hopt_bytes.argtypes = [ct.c_void_p, ct.c_uint32, ct.POINTER(ct.c_uint64)]
        L.hopt_valid.argtypes = [ct.c_void_p, ct.c_uint32, ct.POINTER(ct.c_uint32)]
        L.hopt_write.restype = ct.c_ulonglong
        L.hopt_write.argtypes = [ct.c_uint, ct.c_char_p] + [ct.POINTER(ct.c_void_p)] * 4 + [ct.c_ulonglong, ct.c_uint8, ct.c_uint8,
                                                                                             ct.c_char_p, ct.c_void_p]
        _SO = L
    return _SO


def host_parse(data: bytes, col_types, header=False, null_values=("",)) -> OptParsed:
    L = _shim()
    nulls = (ct.c_char_p * max(1, len(null_values)))(*[s.encode() for s in null_values])
    h = L.hopt_parse(data, len(data), ord(","), ord('"'), int(header), len(col_types), bytes(col_types), len(null_values), nulls)
    cnt = (ct.c_uint32 * 4)()
    L.hopt_counts(h, cnt)
    n_out, n_rows, n_good, n_bad = list(cnt)
    opt = [t & OPT for t in col_types if t != T_SKIP]
    cols, valid = [], []
    for c in range(n_out):
        t = L.hopt_type(h, c)
        if t == T_STR:
            offs = np.ctypeslib.as_array(L.hopt_offsets(h, c), (n_good + 1,)).copy()
            nb = ct.c_uint64()
            p = L.hopt_bytes(h, c, ct.byref(nb))
            cols.append((ct.string_at(p, nb.value) if nb.value else b"", offs))
        else:
            a = np.ctypeslib.as_array(L.hopt_fixed(h, c), (n_good,)).copy().view(np.int64) if n_good else np.zeros(0, np.int64)
            cols.append(a.view(np.float64) if t == T_F64 else a)
        nw = ct.c_uint32()
        p = L.hopt_valid(h, c, ct.byref(nw))
        valid.append((np.ctypeslib.as_array(p, (nw.value,)).copy() if nw.value else np.zeros(0, np.uint32)) if opt[c] else None)
    rowmap = np.ctypeslib.as_array(L.hopt_rowmap(h), (n_good,)).copy() if n_good else np.zeros(0, np.uint32)
    bad = np.ctypeslib.as_array(L.hopt_bad(h), (n_bad * 4,)).copy().reshape(-1, 4) if n_bad else np.zeros((0, 4), np.uint32)
    L.hopt_free(h)
    return OptParsed(n_rows, cols, valid, rowmap, [(int(r[0]), int(r[1])) for r in bad])


def assert_same(a: OptParsed, b: OptParsed, what=""):
    assert a.n_rows == b.n_rows, what
    assert np.array_equal(np.asarray(a.rowmap, np.uint32), np.asarray(b.rowmap, np.uint32)), what
    assert a.bad == b.bad, (what, a.bad[:5], b.bad[:5])
    for c, (x, y) in enumerate(zip(a.columns, b.columns)):
        if isinstance(x, tuple):
            assert x[0] == y[0] and np.array_equal(x[1], y[1]), (what, "string column", c)
        else:
            assert np.array_equal(np.asarray(x).view(np.int64), np.asarray(y).view(np.int64)), (what, "values of column", c)
    for c, (x, y) in enumerate(zip(a.valid, b.valid)):
        assert (x is None) == (y is None), (what, c)
        if x is not None:
            assert np.array_equal(np.asarray(x, np.uint32), np.asarray(y, np.uint32)), (what, "validity of column", c)


def present(p: OptParsed, c: int):
    return [bool((int(p.valid[c][r >> 5]) >> (r & 31)) & 1) for r in range(len(p.rowmap))]


def strings(p: OptParsed, c: int):
    b, o = p.columns[c]
    return [b[o[k]:o[k + 1]].decode() for k in range(len(o) - 1)]


# ---- the reference against hand-derived answers ---------------------------------------------------------------------
@pytest.mark.parametrize("nulls", [[], [""], ["", "NULL"], NULLS_311])
def test_reference_quotednulls(nulls):
    """quotednulls.csv: rows (12, ""), (13, empty), (empty, empty); the quoted `""` dequotes to the empty string."""
    data = golden("quotednulls.csv")
    r = option_reference(data, [T_I64 | OPT, T_STR | OPT], header=True, null_values=nulls)
    assert r.n_rows == 3
    if "" in nulls:
        assert list(r.rowmap) == [0, 1, 2] and not r.bad
        assert list(r.columns[0]) == [12, 13, 0] and present(r, 0) == [True, True, False]
        assert strings(r, 1) == ["", "", ""] and present(r, 1) == [False, False, False]
    else:  # an empty cell is not an i64
        assert list(r.rowmap) == [0, 1] and r.bad == [(2, BADPARSE)]
        assert list(r.columns[0]) == [12, 13] and present(r, 0) == [True, True]
        assert strings(r, 1) == ["", ""] and present(r, 1) == [True, True]
    # the same file without the Option flag: every empty cell makes a NULLERROR row when "" is a null value
    s = option_reference(data, [T_I64, T_STR], header=True, null_values=nulls)
    assert s.bad == ([(0, NULLERROR), (1, NULLERROR), (2, NULLERROR)] if "" in nulls else [(2, BADPARSE)])


@pytest.mark.parametrize("nulls", [[], [""], ["", "NULL"], NULLS_311])
def test_reference_optional_str_test(nulls):
    """optional_str_test.csv: 8 rows of two str columns, empty in one, both or neither."""
    data = golden("optional_str_test.csv")
    cells = [("", ""), ("", ""), ("", "abc"), ("", "abc"), ("abc", ""), ("abc", ""), ("abc", "abc"), ("abc", "abc")]
    r = option_reference(data, [T_STR | OPT, T_STR | OPT], header=False, null_values=nulls)
    assert r.n_rows == 8 and not r.bad and list(r.rowmap) == list(range(8))
    for c in range(2):
        assert present(r, c) == [row[c] not in nulls for row in cells]
        assert strings(r, c) == [row[c] for row in cells]


def test_reference_quoted_nulls_conversion_error_and_cell_count():
    data = b'"NA",1\n"",2\nx,3\n5,""\n7\n"8",4,9\n'
    r = option_reference(data, [T_I64 | OPT, T_I64 | OPT], null_values=["NA", ""])
    assert list(r.rowmap) == [0, 1, 3]
    assert r.bad == [(2, BADPARSE), (4, BADPARSE), (5, BADPARSE)]  # "x" does not convert; 1 and 3 cells for 2 columns
    assert present(r, 0) == [False, False, True] and list(r.columns[0]) == [0, 0, 5]
    assert present(r, 1) == [True, True, False] and list(r.columns[1]) == [1, 2, 0]
    s = option_reference(data, [T_I64, T_I64 | OPT], null_values=["NA", ""])
    assert s.bad[:2] == [(0, NULLERROR), (1, NULLERROR)]


# ---- csvops.cuh built for the host against the reference -------------------------------------------------------------
@pytest.mark.parametrize("name,nulls", [("quotednulls.csv", []), ("quotednulls.csv", [""]), ("optional_str_test.csv", ["", "NULL"]),
                                        ("optional_str_test.csv", NULLS_311)])
def test_host_build_on_fixtures(name, nulls):
    data = golden(name)
    types = [T_I64 | OPT, T_STR | OPT] if name == "quotednulls.csv" else [T_STR | OPT, T_STR]
    header = name == "quotednulls.csv"
    assert_same(host_parse(data, types, header, nulls), option_reference(data, types, header, nulls), name)


def _with_nulls(rng, data: bytes, nulls) -> bytes:
    """Replace a random share of the cells by null values (some quoted)."""
    if not nulls:
        return data
    dens = rng.choice([0.0, 0.05, 0.3, 0.9, 1.0])
    out = []
    for line in data.split(b"\n"):
        cells = line.split(b",")
        for k in range(len(cells)):
            if b'"' not in cells[k] and rng.random() < dens:
                v = rng.choice(nulls).encode()
                cells[k] = b'"' + v + b'"' if rng.random() < 0.2 else v
        out.append(b",".join(cells))
    return b"\n".join(out)


def test_host_build_fuzz():
    rng = random.Random(2024)
    pool = ["", "NULL", "NA", "N/A", "0", "NO CLUE", "Unspecified", "-"]
    for it in range(160):
        ncols = rng.randint(1, 6)
        types = [rng.choice([T_I64, T_F64, T_BOOL, T_STR]) for _ in range(ncols)]
        nulls = rng.sample(pool, rng.randint(0, 8))
        data = gen_csv(rng, rng.randint(0, 120), types, dirty=rng.choice([0.0, 0.05]), weird_quotes=rng.choice([0.0, 0.0, 0.02]))
        data = _with_nulls(rng, data, nulls)
        sel = [(t | OPT) if rng.random() < 0.7 else t for t in types]
        if rng.random() < 0.3:
            sel[rng.randrange(ncols)] = T_SKIP
        header = rng.random() < 0.3
        assert_same(host_parse(data, sel, header, nulls), option_reference(data, sel, header, nulls), f"iteration {it}")


def test_host_sink_writes_none_cells():
    """K7's row writer over validity words: a None cell is the null value quoted once, other cells as before."""
    L = _shim()
    from tuplex_b200.backend import Column
    from tuplex_b200.dataset import _csv_cell
    rows = [(1, "a", None), (None, 'x"y', 2.5), (3, None, None)]
    cols = [Column.from_values([r[c] for r in rows], t) for c, t in enumerate([T_I64, T_STR, T_F64])]
    keep, arrs = [], [(ct.c_void_p * 3)() for _ in range(4)]
    for i, c in enumerate(cols):
        d = np.ascontiguousarray(c.data)
        keep.append(d)
        if c.type == T_STR:
            o = np.ascontiguousarray(c.offsets, dtype=np.uint32)
            keep.append(o)
            arrs[1][i], arrs[2][i] = o.ctypes.data, d.ctypes.data
        else:
            arrs[0][i] = d.ctypes.data
        v = np.ascontiguousarray(c.valid, dtype=np.uint32)
        keep.append(v)
        arrs[3][i] = v.ctypes.data
    for nv in ["", "NULL", "a,b", 'q"']:
        n = L.hopt_write(3, bytes([T_I64, T_STR, T_F64]), *arrs, len(rows), ord(","), ord('"'), nv.encode(), None)
        buf = np.zeros(n + 1, dtype=np.uint8)
        L.hopt_write(3, bytes([T_I64, T_STR, T_F64]), *arrs, len(rows), ord(","), ord('"'), nv.encode(), buf.ctypes.data)
        want = "".join(",".join(_csv_cell(v, nv) for v in r) + "\n" for r in rows)
        assert buf[:n].tobytes().decode() == want, nv


# ---- type inference (CSVStatistic::estimate, disableNullColumns) and hints -------------------------------------------
def _types(tmp_path, text: str, **kw):
    import tuplex_b200
    p = tmp_path / "t.csv"
    p.write_text(text)
    ds = tuplex_b200.Context().csv(str(p), **kw)
    return [t | (OPT if c in ds._source.option_cols else 0) for c, t in enumerate(ds._source.types)]


def test_infer_rare_value_many_nulls(tmp_path):
    """CSVStatsTest.cc RareValueManyNulls: 20 empty rows around one `1.0,` -> (Option[f64], Option[str])"""
    text = ",\n" * 10 + "1.0,\n" + ",\n" * 10
    assert _types(tmp_path, text, header=False, null_values=["", "NULL"]) == [T_F64 | OPT, T_STR | OPT]


def test_infer_band_edges():
    rows = lambda n_null, n: [[""] if k < n_null else ["7"] for k in range(n)]  # noqa: E731
    assert cs.infer_types(rows(10, 100), 1, {""}) == [T_I64]            # exactly 10 %: T
    assert cs.infer_types(rows(11, 100), 1, {""}) == [T_I64 | OPT]      # above 10 %: Option[T]
    assert cs.infer_types(rows(90, 100), 1, {""}) == [T_I64 | OPT]      # exactly 90 %: Option[T]
    assert cs.infer_types(rows(99, 100), 1, {""}) == [T_I64 | OPT]
    assert cs.infer_types(rows(100, 100), 1, {""}) == [T_STR | OPT]     # all null: Option[str]
    assert cs.infer_types(rows(0, 100), 1, {""}) == [T_I64]
    assert cs.infer_types(rows(1, 100), 1, {""}) == [T_I64]             # at most 10 %: today's type


def test_type_hints_optional(tmp_path):
    text = "a,b,c\n1,x,2.5\n2,,\n"
    assert _types(tmp_path, text, type_hints={0: typing.Optional[int], "b": typing.Optional[str]})[:2] == [T_I64 | OPT, T_STR | OPT]
    assert _types(tmp_path, text, type_hints={"c": typing.Optional[float], 1: str})[1:] == [T_STR, T_F64 | OPT]
    assert _types(tmp_path, text, type_hints={0: typing.Optional[bool]})[0] == T_BOOL | OPT
    with pytest.raises(TypeError):
        _types(tmp_path, text, type_hints={0: list})


def test_311_sample_inference():
    """In the NYC sample the 17 empty Incident Zip cells (1.7 %) are below the band: the column is not Option unless hinted."""
    data = golden("311_nyc_sample.csv")
    rows = [[c.decode() for c in cells] for cells, _, _ in cs.iter_rows(data, 44, 34)]
    zi = rows[0].index("Incident Zip")
    types = cs.infer_types(rows[1:], len(rows[0]), {""})
    assert sum(1 for r in rows[1:] if r[zi] == "") == 17 and not types[zi] & OPT


# ---- projection keeps each Option column with its companion ----------------------------------------------------------
_PROJ = {  # Option column k, Option column `other`, and c5 read by the map
    "start": (0, 3, lambda x: (x["c5"] + 1, x["c0"] is None, x["c3"])),
    "middle": (6, 9, lambda x: (x["c5"] + 1, x["c6"] is None, x["c9"])),
    "end": (11, 3, lambda x: (x["c5"] + 1, x["c11"] is None, x["c3"])),
}


@pytest.mark.parametrize("where", ["start", "middle", "end"])
def test_projection_keeps_companions(tmp_path, where):
    """12 file columns, a map reading c5 and two Option columns: the plan decodes those three, the companions follow them in
    the order of their columns, and the loads name the renumbered columns (checked on the plan, nothing runs)."""
    import tuplex_b200
    k, other, udf = _PROJ[where]
    names = [f"c{i}" for i in range(12)]
    p = tmp_path / "w.csv"
    p.write_text(",".join(names) + "\n" + ",".join(str(i) for i in range(12)) + "\n")
    src = tuplex_b200.Context().csv(str(p), type_hints={names[k]: typing.Optional[str], other: typing.Optional[int]})._source
    assert sorted(src.option_cols) == sorted([k, other])
    plan = _compile_stage(src, [Op("map", udf)], None)
    used = sorted({5, k, other})
    assert plan.used_cols == used
    prog, phys, comps = plan.prog, len(used), sorted([k, other])
    assert prog.in_types == [src.types[c] for c in used] + [T_BOOL] * 2
    assert prog.null_of == {phys + m: used.index(c) for m, c in enumerate(comps)}
    loads = {int(i.imm) for i in prog.instrs if i.op == ir.C["TPLX_OP_LDCOL"]}
    assert loads <= set(range(phys + 2))
    assert {used.index(5), phys + comps.index(k)} <= loads  # c5's value and k's "is None" companion
    assert other in src.option_cols and used.index(other) in loads  # `other` flows to the output with its companion
    hdr = prog.serialize()[48:48 + len(prog.in_types)]
    assert list(hdr[phys:]) == [ir.C["TPLX_T_NULLOF"] | used.index(c) for c in comps]


# ---- rows that take the interpreter path ------------------------------------------------------------------------------
def test_line_object_and_host_source_decode_nulls_as_none(tmp_path):
    """Rows whose UDF raised on the device are decoded as the device decoded them: null cells of Option columns are None; a
    null cell in a column that is not Option, or a cell that does not convert, still makes a fallback row."""
    import tuplex_b200
    p = tmp_path / "n.csv"
    p.write_text('a,b,c\n1,"NA",x\n,y,2.5\n3,z,NA\n4,"",\nq,w,1.0\n')
    src = tuplex_b200.Context().csv(str(p), null_values=["", "NA"], type_hints={0: typing.Optional[int], 1: typing.Optional[str],
                                                                                  2: float})._source
    assert src.option_cols == [0, 1]
    assert src.line_object(b'1,"NA",x', True) == (1, None, None)  # x is not an f64
    assert src.line_object(b",y,2.5", True) == (None, "y", 2.5)
    assert src.line_object(b'4,"",1', True) == (4, None, 1.0)
    assert src.line_object(b",w,2.5", False) == (None, "w", 2.5)  # `parse` of the fallback code
    hs = src.to_host_source()
    assert hs.n_rows == 1 and [c.to_values() for c in hs.cols] == [[None], ["y"], [2.5]]
    assert [i for i, _ in hs.fallback] == [0, 2, 3, 4] and hs.cols[0].valid is not None


def test_311_sf1_reads_as_one_option_column(tmp_path):
    """runtuplex.py's csv() call on the one-column sf=1 file: no delimiter to sniff (',' then), the hint makes it Option[str]."""
    import tuplex_b200
    p = tmp_path / "sf1.csv"
    p.write_bytes(golden("311-service-requests-sf=1.csv"))
    src = tuplex_b200.Context().csv(str(p), null_values=NULLS_311, type_hints={0: typing.Optional[str]})._source
    assert src.delimiter == "," and src.names == ["Incident Zip"] and src.types == [T_STR] and src.option_cols == [0]
