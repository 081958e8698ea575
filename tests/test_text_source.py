"""Context.text's device source without a device: the host build of K10's per-line logic (textops.cuh via tests/text_host.cpp)
fuzzed against the host reader (textsource.read_lines), the UTF-8 replacement against CPython, planning (types, columns, cost,
Option flag, degenerate inputs), and the named departures from the reference's TextReader."""
import ctypes as ct
import gzip
import itertools
import os
import random
import subprocess
import typing

import numpy as np
import pytest

import tuplex_b200 as tuplex
from tuplex_b200 import textsource
from tuplex_b200.textsource import TextSource, read_lines

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("text_host") / "text_host.so")
    subprocess.check_call(["g++", "-O1", "-x", "c++", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "text_host.cpp")])
    L = ct.CDLL(so)
    vp, u32, u64 = ct.c_void_p, ct.c_uint32, ct.c_uint64
    L.htext_parse.argtypes = [ct.c_char_p, u32, u32, ct.POINTER(ct.c_char_p), ct.c_int]
    L.htext_parse.restype = vp
    L.htext_counts.argtypes = [vp, ct.POINTER(u64)]
    for f in ("htext_ends", "htext_offsets", "htext_valid", "htext_rowmap", "htext_bad"):
        getattr(L, f).argtypes = [vp]
        getattr(L, f).restype = ct.POINTER(u32)
    L.htext_bytes.argtypes = [vp]
    L.htext_bytes.restype = ct.POINTER(ct.c_uint8)
    L.htext_free.argtypes = [vp]
    L.htext_replace.argtypes = [ct.c_char_p, u32, vp]
    L.htext_replace.restype = u64
    return L


def host_parse(L, data: bytes, nulls=(), option=False):
    """(offsets, bytes, validity words, bad rows) of the host-built K10 pipeline."""
    nv = (ct.c_char_p * max(1, len(nulls)))(*[s.encode() for s in nulls])
    h = L.htext_parse(data, len(data), len(nulls), nv, int(option))
    c = (ct.c_uint64 * 5)()
    L.htext_counts(h, c)
    n_good, n_bad, nb, nw = int(c[1]), int(c[2]), int(c[3]), int(c[4])
    offs = np.ctypeslib.as_array(L.htext_offsets(h), (n_good + 1,)).copy()
    byts = bytes(np.ctypeslib.as_array(L.htext_bytes(h), (nb,))) if nb else b""
    valid = np.ctypeslib.as_array(L.htext_valid(h), (nw,)).copy() if nw else np.zeros(0, np.uint32)
    bad = np.ctypeslib.as_array(L.htext_bad(h), (n_bad * 4,)).reshape(-1, 4).copy() if n_bad else np.zeros((0, 4), np.uint32)
    L.htext_free(h)
    return offs, byts, valid, bad


def expected_block(lines, nulls=(), option=False):
    """The encoded column the host reader's lines give: what _source_from_rows builds (offsets, bytes, validity words in
    block row order), and the null lines that become fallback rows without Option columns."""
    offs, chunks, bits, bad = [0], [], [], []
    for i, ln in enumerate(lines):
        null = ln in nulls
        if null and not option:
            bad.append(i)
            continue
        b = b"" if null else ln.encode()
        chunks.append(b)
        offs.append(offs[-1] + len(b))
        bits.append(not null)
    words = np.zeros((len(bits) + 31) // 32 if (option and nulls) else 0, np.uint32)
    for r, ok in enumerate(bits):
        if ok and len(words):
            words[r // 32] |= np.uint32(1 << (r % 32))
    return np.asarray(offs, np.uint32), b"".join(chunks), words, bad


def lines_of(data: bytes, tmp_path, name="f.txt"):
    p = tmp_path / name
    p.write_bytes(data)
    return read_lines([str(p)], lambda m: None)


def check(L, data, tmp_path, nulls=(), option=False):
    lines = lines_of(data, tmp_path)
    offs, byts, valid, bad = host_parse(L, data, nulls, option)
    eo, eb, ev, ebad = expected_block(lines, nulls, option)
    assert offs.tolist() == eo.tolist()
    assert byts == eb
    assert valid.tolist() == ev.tolist()
    assert bad[:, 0].tolist() == ebad and all(int(c) == 50 for c in bad[:, 1])


# ---- fuzz against the host reader -----------------------------------------------------------------------------------------
PIECES = [b"a", b"hello", b"NULL", b"N/A", b"\n", b"\r\n", b"\r", b"\x00", b"", b"\xef\xbb\xbf", b"\xc3\xa9", b"\xe2\x82\xac",
          b"\xf0\x9f\x98\x80", b"\xff", b"\xe2\x82", b"\xf0\x9f", b"\xed\xa0\x80", b"\xc0\xaf", b"\xef\xbf\xbd", b"x" * 70, b" "]
NULL_SETS = [[], [""], ["NULL", "N/A"], ["", "NULL", "é"], ["�", "a�"], ["€", "😀", ""]]


@pytest.mark.parametrize("seed", range(40))
def test_fuzz_against_host_reader(host, tmp_path, seed):
    rng = random.Random(seed)
    for _ in range(12):
        data = b"".join(rng.choice(PIECES) for _ in range(rng.randrange(0, 400 if seed % 4 else 20000)))
        if rng.random() < 0.3:
            data = data.rstrip(b"\n")  # no final newline
        if rng.random() < 0.2:
            data += b"\r"  # '\r' at EOF
        nulls = rng.choice(NULL_SETS)
        check(host, data, tmp_path, nulls, option=rng.random() < 0.5)


def test_lines_across_tiles(host, tmp_path):
    """Lines spanning 16 KB tiles, one invalid byte in the second tile only (per-tile ASCII flags), sizes tile - 1 .. tile + 1."""
    for n in (16383, 16384, 16385, 3 * 16384 + 7):
        for cut in (0, 1, 63, 64, 16383):
            body = bytearray(b"q" * n)
            for k in range(cut, n, 4097):
                body[k] = 10
            if n > 20000:
                body[20000] = 0xFF
            check(host, bytes(body), tmp_path, ["q" * 5], option=True)


# ---- the replacement against CPython --------------------------------------------------------------------------------------
def _replace_all(L, strings):
    out = []
    buf = ct.create_string_buffer(64)
    for s in strings:
        n = L.htext_replace(s, len(s), buf)
        out.append(buf.raw[:n])
    return out


def test_replacement_exhaustive_one_and_two_bytes(host):
    strings = [bytes([a]) for a in range(256)] + [bytes([a, b]) for a in range(256) for b in range(256)]
    got = _replace_all(host, strings)
    assert got == [s.decode("utf-8", "replace").encode() for s in strings]


def test_replacement_exhaustive_three_bytes(host):
    """All 2^24 three-byte strings, 65536 at a time: each piece is replaced on its own here and written followed by 'A'; CPython
    decodes the same pieces joined by 'A' as one buffer. ASCII ends every sequence in both decoders, so equal output means every
    piece agrees."""
    host.htext_replace_pieces.argtypes = [ct.c_char_p, ct.c_uint64, ct.c_uint32, ct.c_uint32, ct.c_uint8, ct.c_void_p]
    host.htext_replace_pieces.restype = ct.c_uint64
    out = ct.create_string_buffer(65536 * 10)
    bc = np.arange(65536, dtype=np.uint32)
    for a in range(256):
        pieces = np.stack([np.full(65536, a, np.uint8), (bc >> 8).astype(np.uint8), (bc & 255).astype(np.uint8),
                           np.full(65536, ord("A"), np.uint8)], axis=1).tobytes()
        n = host.htext_replace_pieces(pieces, 65536, 3, 4, ord("A"), out)
        assert out.raw[:n] == pieces.decode("utf-8", "replace").encode(), f"lead byte {a:#x}"


def test_replacement_four_bytes(host):
    edges = [0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0]
    strings = [bytes([a, b, c, d]) for a in range(0xF0, 0xF5) for b, c, d in itertools.product(edges, repeat=3)]
    assert _replace_all(host, strings) == [s.decode("utf-8", "replace").encode() for s in strings]


def test_truncated_sequences_at_line_end_and_eof(host, tmp_path):
    for t in (b"\xc3", b"\xe2\x82", b"\xf0\x9f\x98", b"\xf4\x8f\xbf", b"\xe0\xa0", b"\xed\x9f"):
        for data in (t + b"\n" + t, t + b"\r\n" + t + b"\r", b"x" + t, t):
            check(host, data, tmp_path, ["�", "x�"], option=True)
            check(host, data, tmp_path, ["�"], option=False)


# ---- named departures from the reference's TextReader.cc ------------------------------------------------------------------
def test_departure_lone_cr_at_eof_is_stripped(host, tmp_path):
    """TextReader keeps a '\\r' that ends the file without a newline; Context.text strips it like any trailing '\\r'."""
    assert lines_of(b"a\nb\r", tmp_path) == ["a", "b"]
    check(host, b"a\nb\r", tmp_path)
    check(host, b"\r", tmp_path, [""], option=True)


def test_departure_nul_does_not_hide_a_newline(host, tmp_path):
    """TextReader finds newlines with an implicit-length _mm_cmpistri, so a NUL ends its 16-byte window and can merge two lines;
    here a NUL is content."""
    data = b"ab\x00cd\nef\x00\x00\x00\x00\x00\x00\x00\x00\x00\ngh"
    assert lines_of(data, tmp_path) == ["ab\x00cd", "ef" + "\x00" * 9, "gh"]
    check(host, data, tmp_path)


def test_departure_invalid_utf8_is_replaced(host, tmp_path):
    """TextReader hands the raw bytes on; Context.text stores bytes.decode("utf-8", "replace")."""
    assert lines_of(b"a\xffb\n\xe2\x82", tmp_path) == ["a�b", "�"]
    offs, byts, _, _ = host_parse(host, b"a\xffb\n\xe2\x82")
    assert byts == "a�b�".encode() and offs.tolist() == [0, 5, 8]


# ---- planning without a device --------------------------------------------------------------------------------------------
def _write(tmp_path, name, data: bytes):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


@pytest.mark.parametrize("option", ["true", "false"])
def test_planning(tmp_path, option):
    c = tuplex.Context(conf={"tuplex.gpu.optionColumns": option})
    f = _write(tmp_path, "a.txt", b"hello\nNULL\n\nworld\r\nx\xff")
    ds = c.text(f, null_values=["NULL"])
    assert isinstance(ds._source, TextSource) and ds.columns == [None] and ds._cost() == 5
    assert ds.types == ([typing.Optional[str]] if option == "true" else [str])
    assert ds._source.cols[0].to_values() == ["hello", None, "", "world", "x�"]
    assert ds.map(lambda x: len(x)).types == [int]
    plain = c.text(f)  # no null values: a plain str column
    assert isinstance(plain._source, TextSource) and plain.types == [str] and plain._source.option_cols == []
    no_null = c.text(f, null_values=["zzz"])
    assert no_null.types == [str] and no_null._source.option_cols == []
    host = no_null._source.to_host_source()
    assert host.cols[0].to_values() == read_lines([f], print) and host.total_rows == 5


def test_planning_degenerate_inputs_keep_the_host_source(tmp_path):
    c = tuplex.Context()
    empty = _write(tmp_path, "empty.txt", b"")
    nulls = _write(tmp_path, "nulls.txt", b"NULL\r\nNULL\n")
    for ds, n in ((c.text(empty), 0), (c.text(nulls, null_values=["NULL"]), 2), (c.text(str(tmp_path / "missing.txt")), 0),
                  (c.text(nulls, null_values=[str(k) for k in range(9)]), 2)):
        assert not isinstance(ds._source, TextSource) and ds._cost() == n
    assert c.text(nulls, null_values=["NULL"]).types == [typing.Optional[int]]  # today's typing of an all-None column
    assert c.text(nulls, null_values=["x" * 65]).types == [str]  # null values beyond 64 bytes: host source


def test_planning_multiple_files(tmp_path):
    c = tuplex.Context()
    a = _write(tmp_path, "p1.txt", b"b1\nb2")
    b = _write(tmp_path, "p0.txt", b"a1\r\n\n")
    ds = c.text(str(tmp_path / "p*.txt") + "," + str(tmp_path / "nope.txt"))
    assert isinstance(ds._source, TextSource) and ds._cost() == 4
    assert ds._source.cols[0].to_values() == ["a1", "", "b1", "b2"] == read_lines(sorted([a, b]), print)
    assert ds._source.files == sorted([a, b])


def test_count_null_lines_matches_the_reader(tmp_path):
    rng = random.Random(7)
    for _ in range(60):
        data = b"".join(rng.choice(PIECES) for _ in range(rng.randrange(0, 300)))
        nulls = rng.choice(NULL_SETS)
        want = sum(ln in nulls for ln in lines_of(data, tmp_path))
        arr = np.frombuffer(data, np.uint8)
        assert textsource.count_null_lines(arr, [v.encode() for v in nulls]) == want
        assert textsource.count_lines(arr) == len(lines_of(data, tmp_path))


def test_chunks_cut_after_a_newline(tmp_path):
    c = tuplex.Context()
    data = b"".join(b"line%d\n" % i for i in range(1000)) + b"tail"
    ds = c.text(_write(tmp_path, "c.txt", data))
    ds._source.chunk_bytes = 100
    parts = [bytes(a) for a, _ in ds._source.chunks()]
    assert b"".join(parts) == data and all(p.endswith(b"\n") for p in parts[:-1]) and all(len(p) <= 100 for p in parts)


def test_golden_logs_fixture_reads_like_the_reference_file():
    data = gzip.open(os.path.join(HERE, "golden", "logs.sample.txt.gz"), "rb").read()
    assert len(data) == 308807 and textsource.count_lines(np.frombuffer(data, np.uint8)) == 3455
