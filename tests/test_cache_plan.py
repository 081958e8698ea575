"""DataSet.cache() on the device, without a device: the column flags against Context._source_from_rows (the typing the host path
gives the same rows), the re-blocking plan against a cumulative-sum model, and the host build of the UTF-8 rewrite (cache.cuh via
tests/cache_host.cpp) against CPython's decode("utf-8", "replace").encode()."""
import ctypes as ct
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

import tuplex_b200
from tuplex_b200 import backend, dataset
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR

HERE = os.path.dirname(os.path.abspath(__file__))


# ---- column flags ------------------------------------------------------------------------------------------------------------
def _value(rng, t):
    if t == T_I64:
        return rng.randint(-(1 << 63), (1 << 63) - 1)
    if t == T_F64:
        return rng.uniform(-1e9, 1e9)
    if t == T_BOOL:
        return rng.random() < 0.5
    return "".join(rng.choice("abé中,") for _ in range(rng.randint(0, 5)))


@pytest.mark.parametrize("seed", range(40))
def test_flags_type_like_source_from_rows(seed):
    rng = random.Random(seed)
    n = rng.choice([1, 2, 3, 31, 32, 33, 100])
    ncols = rng.choice([1, 1, 2, 5])
    types = [rng.choice([T_I64, T_F64, T_BOOL, T_STR]) for _ in range(ncols)]
    kinds = [rng.choice(["none", "some", "all"]) for _ in range(ncols)]
    cols = []
    for t, kind in zip(types, kinds):
        if kind == "some" and n > 1:
            nones = set(rng.sample(range(n), rng.randint(1, n - 1)))
        else:
            nones = set(range(n)) if kind == "all" else set()
        cols.append([None if i in nones else _value(rng, t) for i in range(n)])
    rows = cols[0] if ncols == 1 else list(zip(*cols))
    src = tuplex_b200.Context()._source_from_rows(rows, None)
    assert not src.fallback and len(src.cols) == ncols
    none_rows = [sum(v is None for v in c) for c in cols]
    invalid = [rng.randint(0, 2) for _ in cols]
    flags = dataset._cache_flags(types, none_rows, invalid, n)
    assert [(t, opt) for _, t, opt in flags] == [(c.type, c.valid is not None) for c in src.cols]
    for (f, t, opt), st, k, bad in zip(flags, types, none_rows, invalid):
        assert bool(f & backend.CONCAT_ALL_NONE) == (k == n)
        assert bool(f & backend.CONCAT_DROP_VALID) == (k == 0)
        assert bool(f & backend.CONCAT_UTF8) == (st == T_STR and bad > 0 and k < n)


# ---- re-blocking plan ----------------------------------------------------------------------------------------------------------
def _model(sizes, B):
    """Every row as (part, row in part), cut into runs of B rows."""
    flat = [(p, r) for p, n in enumerate(sizes) for r in range(n)]
    return [flat[k:k + B] for k in range(0, len(flat), B)]


@pytest.mark.parametrize("seed", range(60))
def test_plan_cuts_at_multiples_of_block_rows(seed):
    rng = random.Random(seed)
    sizes = [rng.choice([0, 0, 1, 2, 5, 31, 32, 33, 64, 100]) for _ in range(rng.randint(0, 8))]
    B = rng.choice([1, 2, 3, 7, 32, 33, 64, 1000])
    plan = dataset._cache_plan(sizes, B)
    want = _model(sizes, B)
    assert len(plan) == len(want)
    for pieces, rows in zip(plan, want):
        assert all(n > 0 for _, _, n in pieces)
        assert [(p, f + k) for p, f, n in pieces for k in range(n)] == rows
        assert len({p for p, _, _ in pieces}) == len(pieces)  # one piece per part and block


def test_plan_edges():
    assert dataset._cache_plan([], 4) == []
    assert dataset._cache_plan([0, 0], 4) == []
    assert dataset._cache_plan([4, 4], 4) == [[(0, 0, 4)], [(1, 0, 4)]]
    assert dataset._cache_plan([3, 0, 6], 4) == [[(0, 0, 3), (2, 0, 1)], [(2, 1, 4)], [(2, 5, 1)]]


# ---- the UTF-8 rewrite ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cache_host") / "cache_host.so")
    subprocess.check_call(["g++", "-O1", "-x", "c++", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "cache_host.cpp")])
    L = ct.CDLL(so)
    L.hcache_rewrite.argtypes = [ct.c_void_p, ct.c_void_p, ct.c_uint64, ct.c_void_p, ct.c_void_p, ct.POINTER(ct.c_uint64)]
    L.hcache_rewrite.restype = ct.c_uint64
    return L


def _rewrite(L, strings):
    data = np.frombuffer(b"".join(strings) + b"\0" * 16, np.uint8)  # the device buffers are readable past their end
    offs = np.zeros(len(strings) + 1, np.uint32)
    np.cumsum([len(s) for s in strings], out=offs[1:])
    out_offs = np.zeros(len(strings) + 1, np.uint32)
    bad = ct.c_uint64()
    total = L.hcache_rewrite(data.ctypes.data, offs.ctypes.data, len(strings), out_offs.ctypes.data, None, ct.byref(bad))
    out = np.zeros(max(total, 1), np.uint8)
    L.hcache_rewrite(data.ctypes.data, offs.ctypes.data, len(strings), out_offs.ctypes.data, out.ctypes.data, ct.byref(bad))
    raw = out[:total].tobytes()
    return [raw[out_offs[i]:out_offs[i + 1]] for i in range(len(strings))], int(bad.value)


def _cpython(b: bytes) -> bytes:
    return b.decode("utf-8", "replace").encode()


def test_rewrite_every_short_string(host):
    """Every 1- and 2-byte string and every 3-byte string over boundary bytes, packed into one column."""
    edge = [0x00, 0x41, 0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0, 0xC1, 0xC2, 0xDF, 0xE0, 0xE1, 0xEC, 0xED, 0xEE, 0xEF,
            0xF0, 0xF1, 0xF3, 0xF4, 0xF5, 0xFF]
    strings = [bytes([a]) for a in range(256)] + [bytes([a, b]) for a in range(256) for b in range(256)]
    strings += [bytes(t) for t in itertools.product(edge, repeat=3)]
    got, bad = _rewrite(host, strings)
    want = [_cpython(s) for s in strings]
    assert got == want
    assert bad == sum(w != s for s, w in zip(strings, want))


def test_rewrite_cut_sequences_nuls_and_empty(host):
    """Multi-byte characters cut at string ends (as a byte slice leaves them), NULs, 0-length strings, long valid strings."""
    rng = random.Random(5)
    text = "aé中\U0001F600z\0".encode()
    strings = [b"", b"\0", b"\0\0abc\0"]
    for _ in range(3000):
        i, j = sorted(rng.randint(0, len(text)) for _ in range(2))
        strings.append(text[i:j] * rng.randint(1, 3))
    strings += [b"", "é".encode() * 500, b"\xe4\xb8", b"", b"\xf0\x9f\x98"]
    got, bad = _rewrite(host, strings)
    assert got == [_cpython(s) for s in strings]
    assert bad == sum(_cpython(s) != s for s in strings)
    assert _rewrite(host, [])[0] == []
