"""Option[T] columns at the CSV boundary on the GPU: K6 through the C ABI against the reference of tests/test_csv_option.py
(values, bit-exact validity words, block row -> data row map, rows handed to the interpreter path), the Option UDF corpus over
a CSV file against CPython, the reference's 311 pipeline (benchmarks/311/runtuplex.py) and K7's None cells against the host
writer."""
import csv as pycsv
import inspect
import io
import os
import random
import typing

import numpy as np
import pytest

import tuplex_b200
from tuplex_b200 import backend, frontend
from tuplex_b200.dataset import _csv_cell
from csv_helpers import T_BOOL, T_F64, T_I64, T_SKIP, T_STR, gen_csv
from option_udfs import UDFS
from test_csv_option import NULLS_311, OPT, OptParsed, _with_nulls, assert_same, golden, option_reference

pytestmark = pytest.mark.gpu


def gpu_parse(data: bytes, types, header=False, null_values=("",)):
    """K6 through the C ABI. The validity words are the block's own (tail bits included, tplx_gpu_block_fetch_validity); the values
    are read back through an identity stage."""
    buf = backend.CsvBuffer(0, data)
    p = buf.parse(types, header=header, null_values=list(null_values))
    info = p.info
    sel = [t for t in types if t != T_SKIP]
    base = [t & ~OPT for t in sel]
    opt = [j for j, t in enumerate(sel) if t & OPT]
    cols, valid = [], [p.block.validity(j) for j in range(len(sel))]
    assert [j for j, v in enumerate(valid) if v is not None] == opt
    sc = frontend.StageCompiler(base, [f"c{j}" for j in range(len(sel))], opt)
    sc.add_map(lambda x: x, 100001)
    st = backend.Stage(sc.finish_memory())
    res = st.run(p.block)
    assert int(res.info.n_out_rows) == int(info.n_normal) and int(res.info.n_exceptions) == 0
    n = int(info.n_normal)
    for j, t in enumerate(base):
        col = res.column(j)
        v = res.validity(j) if j in opt else None
        if j in opt:  # the value under a None is no part of the contract: compare the reference's placeholder 0 / "" there
            vals = [x if ok else ("" if t == T_STR else 0) for x, ok in zip(col.to_values(), backend.unpack_valid(v, n))]
            col = backend.Column.from_values(vals, t)
        cols.append((col.data.tobytes(), col.offsets) if t == T_STR else (col.data.view(np.float64) if t == T_F64 else col.data))
        if v is not None:  # the stage's round trip of the bitmap agrees with the block's
            assert np.array_equal(v, valid[j])
    res.free()
    st.close()
    bad = [(int(b["row"]), int(b["code"])) for b in p.bad_rows()]
    out = OptParsed(int(info.n_rows), cols, valid, p.rowmap(), bad)
    seq = int(info.sequential_rows)
    p.free()
    buf.free()
    return out, seq


@pytest.mark.parametrize("t", [T_I64, T_F64, T_BOOL, T_STR])
@pytest.mark.parametrize("n_good", [32 * 40, 32 * 40 + 1, 32 * 40 + 31])
def test_every_option_type_bit_exact(gpu, t, n_good):
    """Every type as Option, block sizes with n_good % 32 in {0, 1, 31} (the tail word), plus a bad row that shifts the map."""
    rng = random.Random(n_good * 7 + t)
    cell = {T_I64: lambda: str(rng.randint(-9999, 9999)), T_F64: lambda: f"{rng.uniform(-1e3, 1e3):.3f}",
            T_BOOL: lambda: rng.choice(["true", "F", "yes"]), T_STR: lambda: rng.choice(["a", "b c", '"x,y"', "zz"])}[t]
    lines = []
    for k in range(n_good):
        lines.append(",".join([rng.choice(["", "NA", '"NA"']) if rng.random() < 0.3 else cell(), str(k)]))
    lines.insert(n_good // 2, "only-one-cell")
    data = ("\n".join(lines) + "\n").encode()
    types = [t | OPT, T_I64]
    got, _ = gpu_parse(data, types, False, ["", "NA"])
    assert len(got.rowmap) == n_good and got.bad == [(n_good // 2, 70)]
    assert_same(got, option_reference(data, types, False, ["", "NA"]), f"type {t}")


@pytest.mark.parametrize("dens", [0.0, 1.0])
def test_blocks_without_none_and_all_none(gpu, dens):
    rng = random.Random(5)
    lines = [",".join(["" if rng.random() < dens else str(k), "NA" if rng.random() < dens else "s%d" % k]) for k in range(1000)]
    data = ("\n".join(lines) + "\n").encode()
    types = [T_I64 | OPT, T_STR | OPT]
    got, _ = gpu_parse(data, types, False, ["", "NA"])
    assert_same(got, option_reference(data, types, False, ["", "NA"]))
    want = 0 if dens else 0xFFFFFFFF
    assert all(int(w) == want for w in got.valid[0][:-1])


def test_tile_boundaries_and_sequential_repair(gpu):
    """Seeded files of ~200 KB (rows across 16 KB tiles) with nulls in every type, header on and off, and stray quotes that
    force the sequential row finder."""
    rng = random.Random(77)
    pool = ["", "NULL", "NA", "N/A", "0", "NO CLUE", "Unspecified", "-"]
    saw_seq = False
    for it in range(8):
        types = [rng.choice([T_I64, T_F64, T_BOOL, T_STR]) for _ in range(rng.randint(2, 6))]
        nulls = rng.sample(pool, rng.randint(1, 8))
        weird = 0.002 if it % 2 else 0.0
        data = _with_nulls(rng, gen_csv(rng, 6000, types, dirty=0.02, weird_quotes=weird), nulls)
        sel = [(t | OPT) if rng.random() < 0.7 else t for t in types]
        header = it % 3 == 0
        got, seq = gpu_parse(data, sel, header, nulls)
        saw_seq |= bool(seq)
        assert_same(got, option_reference(data, sel, header, nulls), f"iteration {it}")
    assert saw_seq


def test_lazy_option_column_is_refused(gpu):
    buf = backend.CsvBuffer(0, b"a,1\n,2\n")
    with pytest.raises(backend.GpuBackendError):
        buf.parse([T_STR | OPT, T_I64], lazy=[0])
    p = buf.parse([T_STR, T_I64], lazy=[0], null_values=[])  # the same column without the flag stays lazy
    assert int(p.info.n_normal) == 2
    p.free()
    buf.free()


# ---- Option UDFs over a CSV file --------------------------------------------------------------------------------------
def _cpython(fn, rows):
    out, exc = [], 0
    for a, b, c, s in rows:
        try:
            out.append(fn({"a": a, "b": b, "c": c, "s": s}))
        except Exception:  # noqa: BLE001
            exc += 1
    return out, exc


@pytest.mark.parametrize("fn", UDFS, ids=[f.__name__ for f in UDFS])
def test_option_udfs_over_csv(gpu, tmp_path, fn):
    rng = random.Random(11)
    rows = [(None if rng.random() < 0.3 else rng.randint(-5, 12), rng.randint(0, 99), None if rng.random() < 0.4 else rng.randint(0, 9),
             None if rng.random() < 0.3 else rng.choice(["abc", "Xa", "zz", "A b"])) for _ in range(3000)]
    bad_line = 1234
    text = "a,b,c,s\n" + "".join(",".join("" if v is None else str(v) for v in r) + "\n" if k != bad_line else "x,1,2,s\n"
                                  for k, r in enumerate(rows))
    rows[bad_line] = ("x", 1, 2, "s")  # a cell-count-correct row whose `a` does not parse: `parse` of the fallback code
    p = tmp_path / "opt.csv"
    p.write_text(text)
    ctx = tuplex_b200.Context()
    hints = {"a": typing.Optional[int], "b": int, "c": typing.Optional[int], "s": typing.Optional[str]}
    ds = ctx.csv(str(p), null_values=[""], type_hints=hints).map(fn)
    got = ds.collect()
    want, exc = _cpython(fn, rows)
    assert got == want
    assert sum(ds.exception_counts.values()) == exc
    # the device decodes only the columns the UDF reads: the row fails to parse when `a` is one of them
    assert ctx.metrics.csv_bad_rows == (1 if "x['a']" in inspect.getsource(fn) else 0)


# ---- the reference's 311 pipeline (benchmarks/311/runtuplex.py:109-117) ----------------------------------------------
def fix_zip_codes(zips):
    if not zips:
        return None
    # Truncate everything to length 5
    s = zips[:5]

    # Set 00000 zip codes to nan
    if s == "00000":
        return None
    else:
        return s


def _cpython_311(data: bytes, nulls):
    """csv module, the null values, fix_zip_codes, then a set."""
    rd = pycsv.reader(io.StringIO(data.decode("utf-8")))
    zi = next(rd).index("Incident Zip")
    return {fix_zip_codes(None if r[zi] in nulls else r[zi]) for r in rd if r}


def _sorted_lines(b: bytes):
    lines = b.decode().split("\n")
    assert lines[-1] == ""
    return sorted(lines[:-1])


def test_311_pipeline_sf1(gpu, tmp_path):
    """The pipeline as runtuplex.py writes it, on the sf=1 file: every row stays on the device; 246 distinct outputs, None
    included; the tocsv file holds them as the host writer formats them."""
    data = golden("311-service-requests-sf=1.csv")
    path = tmp_path / "sf1.csv"
    path.write_bytes(data)
    want = _cpython_311(data, NULLS_311)
    assert len(want) == 246 and None in want
    ctx = tuplex_b200.Context()
    out = str(tmp_path / "out")
    ctx.csv(str(path), null_values=["Unspecified", "NO CLUE", "NA", "N/A", "0", ""], type_hints={0: typing.Optional[str]}) \
        .mapColumn("Incident Zip", fix_zip_codes).unique().tocsv(out)
    assert ctx.metrics.csv_bad_rows == 0 and ctx.metrics.exceptions == 0
    txt = open(os.path.join(out, "part0.csv"), "rb").read()
    assert _sorted_lines(txt) == sorted(["Incident Zip"] + [_csv_cell(v) for v in want])
    ctx = tuplex_b200.Context()
    got = ctx.csv(str(path), null_values=NULLS_311, type_hints={0: typing.Optional[str]}).mapColumn("Incident Zip", fix_zip_codes) \
        .unique().collect()
    assert set(got) == want and len(got) == len(want)
    assert ctx.metrics.csv_bad_rows == 0 and ctx.metrics.exceptions == 0


@pytest.mark.parametrize("hint", [typing.Optional[str], str])
def test_311_nyc_sample(gpu, tmp_path, hint):
    """41 columns with quoted cells. As Optional[str] no row leaves the device; as str (WrapperTest.NYC311) exactly the 17
    empty-zip rows are NULLERROR rows on the interpreter path and still come out as None."""
    data = golden("311_nyc_sample.csv")
    path = tmp_path / "nyc.csv"
    path.write_bytes(data)
    want = _cpython_311(data, NULLS_311)
    ctx = tuplex_b200.Context()
    ds = ctx.csv(str(path), null_values=NULLS_311, type_hints={"Incident Zip": hint})
    ds = ds.mapColumn("Incident Zip", fix_zip_codes).selectColumns(["Incident Zip"]).unique()
    out = str(tmp_path / "out")
    ds.tocsv(out)
    assert ctx.metrics.csv_bad_rows == (0 if hint is not str else 17) and ctx.metrics.exceptions == 0
    txt = open(os.path.join(out, "part0.csv"), "rb").read()
    assert _sorted_lines(txt) == sorted(["Incident Zip"] + [_csv_cell(v) for v in want])
    got = ds.collect()
    assert set(got) == want and len(got) == len(want) and None in want


# ---- K7: None cells -------------------------------------------------------------------------------------------------
def _k7_none(x):
    if x % 7 == 0:
        return None
    if x % 101 == 5:
        return 10 // (x - x)  # ZeroDivisionError on the device; the resolver below makes it None
    return x * 3


@pytest.mark.parametrize("null_value", [None, "NULL", "a,b", 'q"'])
@pytest.mark.parametrize("source,raise_some", [("csv", False), ("columns", False), ("columns", True)])
def test_tocsv_none_cells(gpu, tmp_path, monkeypatch, null_value, source, raise_some):
    """mapColumn (None on some rows) -> tocsv, written by the device (K7) and compared with the host writer `_csv_cell`. With
    raise_some, rows raise on the device, are resolved to None in CPython and go back into their slots on the device (K9) with
    their validity bits. That path needs a column source: a CSV stage's exception rows merge by input row on the host."""
    from tuplex_b200 import dataset
    rng = random.Random(3)
    rows = [(k, rng.choice(["ab", "c,d", 'e"']), round(rng.random(), 4)) for k in range(5000)]
    udf = _k7_none if raise_some else (lambda x: None if x % 7 == 0 else x * 3)
    device_chunks, merges = [], []
    real_merge, real_resolved = dataset._device_merge_csv, backend.Result.merge_resolved

    def spy_merge(*a, **kw):
        out = real_merge(*a, **kw)
        device_chunks.append(out)
        return out

    def spy_resolved(self, *a, **kw):
        merges.append(len(a[1]))
        return real_resolved(self, *a, **kw)
    monkeypatch.setattr(dataset, "_device_merge_csv", spy_merge)
    monkeypatch.setattr(backend.Result, "merge_resolved", spy_resolved)
    ctx = tuplex_b200.Context()
    if source == "csv":
        p = tmp_path / "in.csv"
        p.write_text("k,s,f\n" + "".join(f"{k},{_csv_cell(s)},{fv}\n" for k, s, fv in rows))
        ds = ctx.csv(str(p))
    else:
        ds = ctx.parallelize(rows, columns=["k", "s", "f"])
    ds = ds.mapColumn("k", udf)
    if raise_some:
        ds = ds.resolve(ZeroDivisionError, lambda x: None)
    out = tmp_path / "out.csv"
    ds.tocsv(str(out), null_value=null_value)
    want = "k,s,f\n"
    for k, s, fv in rows:
        v = None if raise_some and k % 101 == 5 and k % 7 else udf(k)
        want += ",".join(_csv_cell(x, null_value) for x in (v, s, fv)) + "\n"
    assert out.read_bytes().decode() == want
    assert len(device_chunks) == 1 and device_chunks[0] is not None  # the device wrote every row
    if raise_some:
        assert sum(merges) == sum(1 for k in range(5000) if k % 101 == 5 and k % 7)  # resolved rows merged on the device
    else:
        assert not merges


def test_result_csv_still_refuses_option_columns(gpu):
    sc = frontend.StageCompiler([T_I64], ["a"], [0])
    sc.add_map(lambda x: x, 100001)
    st = backend.Stage(sc.finish_memory())
    col = backend.Column.from_values([1, None, 3], T_I64)
    res = st.run_host(0, [col], 3)
    assert res.csv_bytes() is None  # tplx_gpu_result_csv: TPLX_E_UNSUPPORTED
    assert res.csv_bytes(null_value="N") == b"1\nN\n3\n"
    res.free()
    st.close()
