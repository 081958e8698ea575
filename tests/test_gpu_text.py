"""Context.text on the GPU (K10): tplx_gpu_text_parse through the C ABI against the host reader's encoded column (offsets,
bytes, validity words, bad rows, row ends) at its size edges, pipelines through Context against the same pipeline over
ctx.parallelize(host lines), and the reference's known answers (TextParser.cc, DataFrameOperations.cc FastPreview, the Apache
log pipelines of FullPipelines.cc)."""
import gzip
import os
import random

import numpy as np
import pytest

import tuplex_b200
from tuplex_b200 import backend, frontend
from tuplex_b200.ir import T_STR
from tuplex_b200.textsource import TextSource, read_lines
from logs_udfs import ParseWithStrip
from test_text_source import PIECES, expected_block

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def gpu_text(data: bytes, nulls=(), option=False):
    """K10 through the C ABI: (offsets, bytes, validity words, bad rows, rowmap, row ends). The column is read back through an
    identity stage (a None is compared as the empty placeholder the block holds); the validity words are the block's own."""
    buf = backend.CsvBuffer(0, data)
    p = buf.parse_text(list(nulls), option)
    info = p.info
    n = int(info.n_normal)
    valid = p.block.validity(0)
    opt = [0] if valid is not None else []
    sc = frontend.StageCompiler([T_STR], ["line"], opt)
    sc.add_map(lambda x: x, 100001)
    st = backend.Stage(sc.finish_memory())
    res = st.run(p.block)
    assert int(res.info.n_out_rows) == n and int(res.info.n_exceptions) == 0
    vals = res.column(0).to_values()
    if opt:  # the value under a None is no part of the contract: compare the block's empty placeholder there
        vals = [v if ok else "" for v, ok in zip(vals, backend.unpack_valid(res.validity(0), n))]
    res.free()
    st.close()
    col = backend.Column.from_values(vals, T_STR)
    offs = col.offsets.astype(np.uint32) if n else np.zeros(1, np.uint32)
    out = (offs, col.data.tobytes()[: int(offs[-1])], valid if valid is not None else np.zeros(0, np.uint32), p.bad_rows(),
           p.rowmap(), p.row_ends(), int(info.n_rows))
    p.free()
    buf.free()
    return out


def check_abi(data: bytes, tmp_path, nulls=(), option=False):
    f = tmp_path / "abi.txt"
    f.write_bytes(data)
    lines = read_lines([str(f)], print)
    offs, byts, valid, bad, rowmap, ends, n_rows = gpu_text(data, nulls, option)
    eo, eb, ev, ebad = expected_block(lines, nulls, option)
    assert n_rows == len(lines)
    assert offs.tolist() == eo.tolist() and byts == eb
    assert valid.tolist() == ev.tolist()
    assert bad["row"].tolist() == ebad and all(int(c) == 50 for c in bad["code"])
    bad_set = set(ebad)
    assert rowmap.tolist() == [i for i in range(len(lines)) if i not in bad_set]
    e = ends.astype(np.int64)
    e[0] = -1
    for i in random.Random(1).sample(range(len(lines)), min(len(lines), 200)):  # the row ends cut every line's bytes
        raw = data[e[i] + 1:e[i + 1]]
        raw = raw[:-1] if raw.endswith(b"\r") else raw
        assert raw.decode("utf-8", "replace") == lines[i]


@pytest.mark.parametrize("data", [b"", b"x", b"x\n", b"\n", b"\r", b"\r\n\r\n", b"a\nb\r", b"\xff\n\xe2\x82"])
def test_abi_tiny(gpu, tmp_path, data):
    for nulls, option in (((), False), (("",), True), (("", "x"), False)):
        check_abi(data, tmp_path, nulls, option)


@pytest.mark.parametrize("size", [16383, 16384, 16385, 2 * 16384 + 1])
def test_abi_tile_edges(gpu, tmp_path, size):
    rng = random.Random(size)
    data = bytearray(rng.choice(b"abc \r\n") for _ in range(size))
    data[size // 2] = 0xE2  # one truncated sequence in one tile
    for nulls, option in (((), False), (("a", ""), True), (("a", "b"), False)):
        check_abi(bytes(data), tmp_path, nulls, option)
        check_abi(bytes(data[:-1]) + b"\n", tmp_path, nulls, option)


def test_abi_many_lines(gpu, tmp_path):
    """More than 2^21 lines: several scan blocks of tiles and of lines."""
    data = b"".join(b"%d\n" % (i % 1000) if i % 97 else b"N\r\n" for i in range((1 << 21) + 12345))
    check_abi(data, tmp_path, ("N",), True)
    check_abi(data, tmp_path, ("N",), False)


def test_abi_long_lines(gpu, tmp_path):
    rng = random.Random(3)
    parts = []
    for ln in (0, 1, 31, 32, 33, 63, 64, 65, 16383, 16384, 16385, 100000, 1 << 20):
        body = bytearray(rng.choice(b"xyz\x00") for _ in range(ln))
        if ln > 40:
            body[ln // 3] = 0xFF  # a replaced line: written by one lane
        parts.append(bytes(body))
        parts.append(bytes(rng.choice(b"pq") for _ in range(ln)))  # a verbatim one: the whole warp
    check_abi(b"\n".join(parts), tmp_path, ("",), True)


def test_abi_fuzz(gpu, tmp_path):
    rng = random.Random(11)
    for _ in range(30):
        data = b"".join(rng.choice(PIECES) for _ in range(rng.randrange(0, 5000)))
        nulls = rng.choice([[], [""], ["NULL", "N/A"], ["�", ""], ["é", "😀"]])
        check_abi(data, tmp_path, nulls, rng.random() < 0.5)


def test_abi_null_value_limits(gpu):
    buf = backend.CsvBuffer(0, b"a\n")
    with pytest.raises(backend.GpuBackendError):
        buf.parse_text([str(k) for k in range(9)])
    with pytest.raises(backend.GpuBackendError):
        buf.parse_text(["x" * 65])
    buf.free()


# ---- through Context ------------------------------------------------------------------------------------------------------
def _ctx(option):
    return tuplex_b200.Context(conf={"tuplex.gpu.optionColumns": option})


def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def _fuzz_text(seed, n):
    rng = random.Random(seed)
    words = ["12", "-7", "abc", "", "NULL", "3.5", "é", "x\x00y", "99", "  4 "]
    out = []
    for _ in range(n):
        w = rng.choice(words)
        out.append(w.encode() + rng.choice([b"\n", b"\r\n"]))
        if rng.random() < 0.01:
            out.append(b"bad\xff\n")
    return b"".join(out)


PIPELINES = {
    "len": lambda ds: ds.map(lambda x: len(x) if x is not None else -1),
    "filter": lambda ds: ds.filter(lambda x: x is not None and len(x) > 2).map(lambda x: x.upper()),
    "int_ignore": lambda ds: ds.map(lambda x: int(x)).ignore(ValueError),
    "int_resolve": lambda ds: ds.map(lambda x: int(x)).resolve(ValueError, lambda x: -1),
    "int_raise": lambda ds: ds.map(lambda x: int(x) * 2),
    "unique": lambda ds: ds.unique(),
    "by_key": lambda ds: ds.map(lambda x: (x if x is not None else "-", 1)).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x[1], 0, [0]),
}


@pytest.mark.parametrize("option", ["true", "false"])
@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_pipelines_match_parallelize(gpu, tmp_path, option, name):
    f1 = _write(tmp_path, "b.txt", _fuzz_text(1, 3000))
    f2 = _write(tmp_path, "a.txt", _fuzz_text(2, 2000) + b"tail")
    for nulls in (None, ["NULL", ""]):
        ctx = _ctx(option)
        ds = ctx.text(str(tmp_path / "*.txt"), null_values=nulls)
        assert isinstance(ds._source, TextSource)
        ds._source.chunk_bytes = 7000  # several chunks per file, each cut after a newline
        got = PIPELINES[name](ds).collect()
        host = [None if (nulls and ln in nulls) else ln for ln in read_lines(sorted([f1, f2]), print)]
        ref_ctx = _ctx(option)
        want = PIPELINES[name](ref_ctx.parallelize(host)).collect()
        assert got == want
        assert ctx.metrics.text_rows == len(host) and not any("falls back" in m for m in ctx._messages)


def test_exception_counts_match(gpu, tmp_path):
    f = _write(tmp_path, "e.txt", _fuzz_text(5, 4000))
    ctx = _ctx("true")
    ds = ctx.text(f).map(lambda x: int(x))
    rows = ds.collect()
    ref = ctx.parallelize(read_lines([f], print)).map(lambda x: int(x))
    assert rows == ref.collect()
    # one map operator on each side; the operator ids differ, the counts per exception class must not
    assert sorted((k[1], v) for k, v in ds.exception_counts.items()) == sorted((k[1], v) for k, v in ref.exception_counts.items())
    assert len(ds.exception_counts) == 1


# ---- the reference's known answers ----------------------------------------------------------------------------------------
def test_textparse_basic(gpu, tmp_path):
    """TextParser.cc TextParse.Basic"""
    ctx = _ctx("true")
    assert ctx.text(_write(tmp_path, "t.txt", b"hello\nhow\n\nis everything?")).collect() == ["hello", "how", "", "is everything?"]
    assert ctx.metrics.text_rows == 4


def test_textparse_null_values(gpu, tmp_path):
    """TextParser.cc TextParse.NULLValues"""
    ctx = _ctx("true")
    f = _write(tmp_path, "t.txt", b"hello\nworld\nNULL\nN/A\ntest\n\nhow is everything?\n")
    assert ctx.text(f, ["", "NULL", "N/A"]).collect() == ["hello", "world", None, None, "test", None, "how is everything?"]
    assert ctx.metrics.text_rows == 7


def test_fast_preview_take(gpu, tmp_path):
    """DataFrameOperations.cc DataFrameTest.FastPreview (text part)"""
    ctx = _ctx("true")
    assert ctx.text(_write(tmp_path, "t.txt", b"A\nB\nC\nD\nE\nF\nG\nH\nI\nJ")).map(lambda x: x.lower()).take(5) == ["a", "b", "c", "d", "e"]


def _golden(tmp_path, name):
    return _write(tmp_path, name, gzip.open(os.path.join(HERE, "golden", name + ".gz"), "rb").read())


def test_apache_dev_join_count(gpu, tmp_path):
    """FullPipelines.cc PipelinesTest.ApacheDev: the logs joined with the bad IPs give 3437 rows (the strip variant)."""
    logs, ips = _golden(tmp_path, "logs.sample.txt"), _golden(tmp_path, "bad_ips_all.txt")
    ctx = _ctx("true")
    rows = ctx.text(logs).map(ParseWithStrip).join(ctx.csv(ips), "ip", "BadIPs").collect()
    bad = [ln for ln in read_lines([ips], print)[1:]]
    want = [r for r in map(ParseWithStrip, read_lines([logs], print)) for b in bad if r["ip"] == b]
    assert len(rows) == len(want) == 3437
    assert ctx.metrics.text_rows > 0 and not any("falls back" in m for m in ctx._messages)


def test_null_value_apache_tocsv(gpu, tmp_path):
    """FullPipelines.cc PipelinesTest.NullValueApache's golden output, over ip_blacklist.csv."""
    logs, ips = _golden(tmp_path, "logs.sample.txt"), _golden(tmp_path, "ip_blacklist.csv")
    ctx = _ctx("true")
    out = str(tmp_path / "logs.csv")
    ctx.text(logs).map(ParseWithStrip).join(ctx.csv(ips), "ip", "BadIPs").selectColumns(["ip", "endpoint"]).tocsv(out)
    assert open(out, "rb").read() == b"ip,endpoint\n1.1.209.108,/research/finance/\n"
    assert ctx.metrics.text_rows > 0 and not any("falls back" in m for m in ctx._messages)
