"""Hash join (K8, csrc/join.cuh) against a plain reference at its key, bucket, collision and size edges.

The reference below is a dict-of-lists join over Python values (numpy's stable argsort + searchsorted for the large cases). It gives
the contract's order: probe rows in input order, each probe row's matches in build-row order. Outputs are compared as raw column
data: the bits of fixed-width values, string bytes and offsets, and the present bits of the validity words.

The join's output does not depend on where keys sit in the table, so the colliding key sets are built on purpose from a Python
restatement of the key hashes (csrc/keyhash.cuh), which the CPU part checks against the header compiled for the host. With them
the GPU part puts keys that differ only in their high 32 bits, or only in their last byte, on one probe chain, and makes chains
wrap from slot cap - 1 to slot 0."""
import ctypes as ct
import functools
from collections import Counter
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from tuplex_b200 import backend, dataset
from tuplex_b200.backend import Column, pack_valid, unpack_valid
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR

HERE = os.path.dirname(os.path.abspath(__file__))
M64 = (1 << 64) - 1
CAP = 1024  # table capacity of every build side up to 512 rows (load <= 0.5)
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
MODES = ["inner", "left", "build_first"]


# ---- the key hashes of csrc/keyhash.cuh, restated ----------------------------------------------------------------------------
def mix64(x):
    x ^= x >> 33
    x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33
    x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x


def hash_i64(v):
    return mix64((v & M64) ^ 0x9E3779B97F4A7C15)


def hash_bytes(b: bytes):
    f = 0xcbf29ce484222325
    for c in b:
        f = ((f ^ c) * 0x100000001b3) & M64
    return mix64(f ^ ((len(b) << 48) & M64))


def home(h, cap=CAP):
    """First slot of a key's probe chain (join_insert_kernel / join_probe_count_kernel)."""
    return (h >> 17) & (cap - 1)


def _np_mix64(x):
    x = x.astype(np.uint64)
    x ^= x >> np.uint64(33)
    x *= np.uint64(0xff51afd7ed558ccd)
    x ^= x >> np.uint64(33)
    x *= np.uint64(0xc4ceb9fe1a85ec53)
    x ^= x >> np.uint64(33)
    return x


def _np_home_i64(v):
    return (_np_mix64(v.astype(np.int64).view(np.uint64) ^ np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(17)) & np.uint64(CAP - 1)


def _np_home_bytes(mat):
    """Home slots of the rows of a (N, L) uint8 matrix, each row one key of L bytes."""
    f = np.full(mat.shape[0], 0xcbf29ce484222325, np.uint64)
    for i in range(mat.shape[1]):
        f = (f ^ mat[:, i].astype(np.uint64)) * np.uint64(0x100000001b3)
    return (_np_mix64(f ^ np.uint64((mat.shape[1] << 48) & M64)) >> np.uint64(17)) & np.uint64(CAP - 1)


def _key_home(v):
    return home(hash_bytes(v) if isinstance(v, bytes) else hash_i64(int(v)))


def _table_slots(distinct_keys):
    """Linear probing of the distinct non-None keys into CAP slots. Which slots end up occupied does not depend on the order of the
    inserts, so this is the layout the device's atomic inserts produce too."""
    occ = np.zeros(CAP, bool)
    for k in distinct_keys:
        i = _key_home(k)
        while occ[i]:
            i = (i + 1) & (CAP - 1)
        occ[i] = True
    return occ


def _walk(occ, slot):
    """Occupied slots a lookup starting at `slot` passes before it reaches an empty one."""
    n = 0
    while occ[slot]:
        n += 1
        slot = (slot + 1) & (CAP - 1)
    return n


# ---- columns -----------------------------------------------------------------------------------------------------------------
def scol(values):
    """String column from bytes (None = Option): the bytes go in as they are, which Column.from_values (UTF-8 text) cannot do."""
    present = [v is not None for v in values]
    enc = [v if v is not None else b"" for v in values]
    offsets = np.zeros(len(enc) + 1, np.uint32)
    np.cumsum([len(e) for e in enc], out=offsets[1:])
    data = np.frombuffer(b"".join(enc), np.uint8).copy()
    return Column(T_STR, data, offsets, None if all(present) else pack_valid(np.array(present, bool)))


def icol(values, t=T_I64):
    present = [v is not None for v in values]
    data = np.array([int(v) if v is not None else 0 for v in values], np.int64)
    return Column(t, data, None, None if all(present) else pack_valid(np.array(present, bool)))


def fcol_bits(bits, present=None):
    return Column(T_F64, np.array(bits, np.uint64).view(np.float64), None, None if present is None or all(present) else pack_valid(np.array(present, bool)))


def key_values(col):
    """Python values of a key column: int, bool, bytes or None."""
    n = len(col)
    pres = np.ones(n, bool) if col.valid is None else unpack_valid(col.valid, n)
    if col.type == T_STR:
        raw, o = col.data.tobytes(), col.offsets
        vals = [raw[int(o[i]):int(o[i + 1])] for i in range(n)]
    elif col.type == T_BOOL:
        vals = [bool(v) for v in col.data.tolist()]
    else:
        vals = col.data.tolist()
    return [v if p else None for v, p in zip(vals, pres.tolist())]


def nrows(cols):
    return len(cols[0])


# ---- the reference -----------------------------------------------------------------------------------------------------------
def _tag(v):
    return None if v is None else (type(v), v)  # keys match only when their types match; None matches None


def ref_pairs_values(build_keys, probe_keys, left_outer):
    """(probe rows, build rows) of the join; build row -1 = a left-joined probe row without a match."""
    table = {}
    for j, v in enumerate(build_keys):
        table.setdefault(_tag(v), []).append(j)
    op, ob = [], []
    for i, v in enumerate(probe_keys):
        ms = table.get(_tag(v), [])
        op += [i] * len(ms)
        ob += ms
        if left_outer and not ms:
            op.append(i)
            ob.append(-1)
    return np.array(op, np.int64), np.array(ob, np.int64)


def ref_pairs(build_key: Column, probe_key: Column, left_outer):
    return ref_pairs_values(key_values(build_key), key_values(probe_key), left_outer)


def ref_pairs_np(build_keys, probe_keys, left_outer):
    """The same join for large i64 key arrays without None: stable argsort of the build keys, then searchsorted."""
    order = np.argsort(build_keys, kind="stable")
    sk = build_keys[order]
    lo = np.searchsorted(sk, probe_keys, "left")
    cnt = np.searchsorted(sk, probe_keys, "right") - lo
    emit = np.where(cnt == 0, 1 if left_outer else 0, cnt)
    op = np.repeat(np.arange(len(probe_keys), dtype=np.int64), emit)
    within = np.arange(op.size, dtype=np.int64) - np.repeat(np.cumsum(emit) - emit, emit)
    miss = np.repeat(cnt == 0, emit)
    ob = order[np.minimum(np.repeat(lo, emit) + within, max(len(order) - 1, 0))] if len(order) else np.zeros(op.size, np.int64)
    return op, np.where(miss, -1, ob).astype(np.int64)


def expected_layout(build, bk, probe, pk, op, ob, mode):
    """(source column, source rows, nullable by the join) per output column: | first side's non-key | key (probe row's) | second
    side's non-key |, the build side first only for build_first."""
    ps = [(c, op, False) for i, c in enumerate(probe) if i != pk]
    bs = [(c, ob, mode == "left") for i, c in enumerate(build) if i != bk]
    key = [(probe[pk], op, False)]
    return bs + key + ps if mode == "build_first" else ps + key + bs


def assert_column(got: Column, src: Column, idx, nullable, what):
    n = len(idx)
    has = idx >= 0
    sidx = np.where(has, idx, 0)
    src_pres = np.ones(len(src), bool) if src.valid is None else unpack_valid(src.valid, len(src))
    pres = has & src_pres[sidx] if len(src) else np.zeros(n, bool)
    assert got.type == src.type, what
    if nullable or src.valid is not None:
        assert got.valid is not None, f"{what}: no validity words"
        assert len(got.valid) == (n + 31) // 32, what
        gp = unpack_valid(got.valid, n)
        bad = np.flatnonzero(gp != pres)
        assert bad.size == 0, f"{what}: present bits differ at rows {bad[:8].tolist()}"
    else:
        assert got.valid is None, f"{what}: unexpected validity words"
    if src.type == T_STR:
        so = src.offsets.astype(np.int64)
        lens = np.where(has, so[sidx + 1] - so[sidx], 0) if len(src) else np.zeros(n, np.int64)
        eo = np.zeros(n + 1, np.int64)
        np.cumsum(lens, out=eo[1:])
        go = got.offsets.astype(np.int64)
        bad = np.flatnonzero(go != eo)
        assert bad.size == 0, f"{what}: string offsets differ from row {bad[:1].tolist()}"
        pos = np.repeat(so[sidx] - eo[:-1], lens) + np.arange(eo[-1], dtype=np.int64)
        exp = src.data[pos] if pos.size else np.zeros(0, np.uint8)
        assert len(got.data) == len(exp), what
        bad = np.flatnonzero(got.data != exp)
        if bad.size:
            row = int(np.searchsorted(eo, bad[0], "right") - 1)
            raise AssertionError(f"{what}: string bytes differ in row {row}: {got.data[eo[row]:eo[row + 1]].tobytes()!r} "
                                 f"vs {exp[eo[row]:eo[row + 1]].tobytes()!r}")
    else:
        gd = np.ascontiguousarray(got.data).view(np.uint64)
        sd = np.ascontiguousarray(src.data).view(np.uint64)
        exp = sd[sidx] if len(src) else np.zeros(n, np.uint64)
        bad = np.flatnonzero(pres & (gd != exp))
        assert bad.size == 0, f"{what}: values differ at rows {bad[:8].tolist()}: {gd[bad[:4]].tolist()} vs {exp[bad[:4]].tolist()}"


def probe_table(j: backend.Join, build, probe, pk, mode):
    pb = backend.Block.upload(0, probe, nrows(probe))
    res = j.probe(pb, [c.type for c in probe], pk, left_outer=mode == "left", build_first=mode == "build_first")
    n_out = int(res.info.n_out_rows)
    got = res.columns()
    res.free()
    pb.free()
    return got, n_out


def check_probe(j, build, bk, probe, pk, mode, pairs=None):
    op, ob = pairs if pairs is not None else ref_pairs(build[bk], probe[pk], mode == "left")
    got, n_out = probe_table(j, build, probe, pk, mode)
    assert n_out == len(op)
    lay = expected_layout(build, bk, probe, pk, op, ob, mode)
    assert len(got) == len(lay)
    for k, (g, (src, idx, nullable)) in enumerate(zip(got, lay)):
        assert_column(g, src, idx, nullable, f"{mode} output column {k}")
    return op, ob


def check_join(build, bk, probe, pk, mode, pairs=None):
    """Build a table over `build`, probe it with `probe`, compare every output column; returns (op, ob, Join.info)."""
    bb = backend.Block.upload(0, build, nrows(build))
    j = backend.Join(bb, [c.type for c in build], bk)
    try:
        op, ob = check_probe(j, build, bk, probe, pk, mode, pairs)
        info = j.info
    finally:
        j.free()
        bb.free()
    return op, ob, info


def with_payloads(keys: Column, tag, key_pos=0):
    """A side of a join: the key column at key_pos among an i64 row id and a string payload that names the row."""
    n = len(keys)
    cols = [icol(range(n)), scol([b"%s%d" % (tag, i) * int(i % 3) for i in range(n)])]
    cols.insert(key_pos, keys)
    return cols


# ---- the small-case matrix (key columns; the GPU part adds payloads) ----------------------------------------------------------
def _spread(rng, keys):
    keys = list(keys)
    rng.shuffle(keys)
    return keys


@functools.lru_cache(maxsize=None)
def colliding_i64():
    """(build keys, probe keys, groups): keys whose chains wrap from slot 1023 to 0, and pairs k, k + m * 2^32 on one chain."""
    cand = np.arange(1, 1 << 21, dtype=np.int64)
    homes = _np_home_i64(cand).astype(np.int64)
    wrap = cand[homes == CAP - 1][:10].tolist()
    wrap_in, wrap_absent = wrap[:6], wrap[6:]
    in_cluster_absent = cand[homes <= 2][:3].tolist()  # misses that start inside the wrapped cluster
    ms = np.arange(-(1 << 15), 1 << 15, dtype=np.int64)
    fam = 0x5EED + (ms << np.int64(32))  # one low 32-bit word, 65536 high words
    fam_homes = _np_home_i64(fam).astype(np.int64)
    pairs, pair_absent = [], []
    for s in range(16, 20):
        members = fam[fam_homes == s].tolist()  # ascending: the first is negative, the last positive
        pairs.append([members[0], members[-1]])
        pair_absent.append(members[1])
    rng = np.random.default_rng(1)
    filler = rng.integers(-(1 << 62), 1 << 62, 60).tolist()
    distinct = wrap_in + [k for p in pairs for k in p] + filler
    build = _spread(rng, [k for i, k in enumerate(distinct) for _ in range(1 + i % 3)])
    probe = _spread(rng, distinct + distinct[:20] + wrap_absent + pair_absent + in_cluster_absent)
    return build, probe, {"wrap": wrap_in, "wrap_absent": wrap_absent, "pairs": pairs, "pair_absent": pair_absent,
                          "cluster_absent": in_cluster_absent}


@functools.lru_cache(maxsize=None)
def colliding_str():
    """Strings on one chain that differ only in their last byte, or only in length (p vs p + b"\\0"), and a chain across slot 1023."""
    rng = np.random.default_rng(2)
    wrap, n = [], 0
    while len(wrap) < 7:
        s = b"w%d" % n
        if _key_home(s) == CAP - 1:
            wrap.append(s)
        n += 1
    wrap_in, wrap_absent = wrap[:4], wrap[4:]
    pairs, pair_absent = [], []
    for plen in (0, 1, 2, 6, 15, 16, 30, 63, 128, 255, 256):
        prefix = rng.integers(0, 256, plen, dtype=np.uint8)
        mat = np.concatenate([np.tile(prefix, (256, 1)), np.arange(256, dtype=np.uint8)[:, None]], axis=1)
        homes = _np_home_bytes(mat).astype(np.int64)
        vals, cnt = np.unique(homes, return_counts=True)
        s = int(vals[np.argmax(cnt)])
        members = [mat[i].tobytes() for i in np.flatnonzero(homes == s)]
        pairs.append(members[:2])
        pair_absent.append(members[2] if len(members) > 2 else bytes(prefix) + bytes([(members[0][-1] + 1) & 0xFF]))
    len_pairs = []
    for width in (2, 8):
        p = np.arange(1 << 16, dtype=np.uint64 if width == 8 else np.uint16).view(np.uint8).reshape(-1, width)
        same = np.flatnonzero(_np_home_bytes(p) == _np_home_bytes(np.concatenate([p, np.zeros((len(p), 1), np.uint8)], axis=1)))
        len_pairs += [[p[i].tobytes(), p[i].tobytes() + b"\0"] for i in same[:2]]
    filler = [rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8).tobytes() for _ in range(60)]
    distinct = wrap_in + [k for p in pairs + len_pairs for k in p] + [b"a", b"a\0"] + filler
    build = _spread(rng, [k for i, k in enumerate(distinct) for _ in range(1 + i % 3)])
    probe = _spread(rng, distinct + distinct[:15] + wrap_absent + pair_absent + [b"a\0\0", b""])
    return build, probe, {"wrap": wrap_in, "wrap_absent": wrap_absent, "pairs": pairs, "pair_absent": pair_absent, "len_pairs": len_pairs}


I64_EDGES = [0, 1, -1, INT64_MIN, INT64_MAX, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, -(1 << 32), 1 << 31, -(1 << 31) - 1, INT64_MIN + 1]
I64_ABSENT = [2, -2, INT64_MAX - 1, (1 << 32) + 2, 1 << 33, -(1 << 32) - 1]


def _str_edge_keys():
    """"" next to None, non-UTF-8 bytes, embedded NULs, lengths 1-257; the columns' lengths put key starts at every offset mod 16."""
    rng = np.random.default_rng(3)
    keys = [b"", None, b"\xff", b"\xc3\x28", b"\x80\x00\x80", b"\0", b"\0\0", b"a\0b", b"\xed\xa0\x80", b"caf\xc3\xa9"]
    for ln in (1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257):
        keys.append(rng.integers(0, 256, ln, dtype=np.uint8).tobytes())
        keys.append(b"x" * ln)
    return keys


@functools.lru_cache(maxsize=None)
def key_value_cases():
    rng = np.random.default_rng(4)
    sk = _str_edge_keys()
    absent_s = [b"\xfe", b"x" * 258, b"\0\0\0", b"caf\xc3\xa9 ", b"\xc3"]
    # 16 keys of 17 bytes in a row: whatever comes before them, they start at every offset mod 16
    tail = [b"%02d" % i + b"\x80\0" * 7 + b"t" for i in range(16)]
    return {
        "i64": (T_I64, _spread(rng, I64_EDGES + I64_EDGES[::2]), _spread(rng, I64_EDGES * 2 + I64_ABSENT)),
        "bool": (T_BOOL, _spread(rng, [True, False, None] * 3 + [True]), [True, None, False, None, True, False]),
        "bool_no_none": (T_BOOL, [False, True, False], [True, False, True, True]),
        "str": (T_STR, _spread(rng, sk + sk[::3]) + tail, _spread(rng, sk + sk[1::2] + absent_s) + tail),
        "str_empty_vs_none": (T_STR, [b"", b"", None, b"z"], [None, b"", b"z", None, b""]),
    }


def _kcol(t, keys):
    return scol(keys) if t == T_STR else icol(keys, t)


@functools.lru_cache(maxsize=None)
def null_cases():
    """Option keys on one side only and on both; null buckets of 0, 1, 33 and 2049 rows; an all-null build side."""
    rng = np.random.default_rng(5)
    out = {}
    for n_null in (0, 1, 33, 2049):
        build = _spread(rng, [None] * n_null + [int(v) for v in rng.integers(0, 50, 300)])
        probe = _spread(rng, [None] * 7 + [int(v) for v in rng.integers(0, 60, 100)])
        out[f"both_{n_null}"] = (T_I64, build, probe)
    out["build_only"] = (T_I64, _spread(rng, [None] * 40 + list(range(30)) * 2), list(range(-5, 35)))
    out["probe_only"] = (T_I64, list(range(30)) * 2, _spread(rng, [None] * 40 + list(range(-5, 35))))
    out["all_null_build"] = (T_I64, [None] * 50, _spread(rng, [None] * 3 + list(range(10))))
    out["str_both"] = (T_STR, _spread(rng, [None] * 33 + [b"k%d" % i for i in range(40)] + [b""] * 3),
                       _spread(rng, [None, None, b"", b"k3", b"k99"] + [b"k%d" % i for i in range(0, 40, 3)]))
    return out


BUCKET_SIZES = [1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4097]


def _warp_mixed_probe(rng, wide, narrow, missing, n_warps):
    """Probe keys in warps of 32 rows, each warp holding wide rows (32+ matches), narrow rows and misses, in shuffled lanes."""
    keys = []
    for _ in range(n_warps):
        w = [wide[int(rng.integers(len(wide)))] if wide else missing[0] for _ in range(int(rng.integers(1, 8)))]
        w += [narrow[int(rng.integers(len(narrow)))] for _ in range(int(rng.integers(4, 16)))]
        w += [missing[int(rng.integers(len(missing)))] for _ in range(32 - len(w))]
        keys += _spread(rng, w)
    return keys + [narrow[0], missing[0]] + ([wide[0]] if wide else [])  # and a partial last warp


@functools.lru_cache(maxsize=None)
def bucket_case(size):
    """One key with `size` build rows spread over the build side among 300 one-row keys."""
    rng = np.random.default_rng(100 + size)
    build = _spread(rng, [7] * size + list(range(1000, 1300)))
    wide = [7] if size >= 32 else []
    narrow = ([7] if size < 32 else []) + list(range(1000, 1300, 7))
    probe = _warp_mixed_probe(rng, wide, narrow, [-1, -2, 5000], 8)
    return build, probe


@functools.lru_cache(maxsize=None)
def all_buckets_case():
    rng = np.random.default_rng(6)
    build = _spread(rng, [k for k, s in enumerate(BUCKET_SIZES) for _ in range(s)])
    wide = [k for k, s in enumerate(BUCKET_SIZES) if s >= 32]
    narrow = [k for k, s in enumerate(BUCKET_SIZES) if s < 32]
    probe = _warp_mixed_probe(rng, wide, narrow, [-7, 100, 1 << 40], 10) + list(range(len(BUCKET_SIZES)))
    return build, probe


def small_key_matrix():
    """Every small case as (name, key type, build keys, probe keys)."""
    out = []
    b, p, _ = colliding_i64()
    out.append(("colliding_i64", T_I64, b, p))
    b, p, _ = colliding_str()
    out.append(("colliding_str", T_STR, b, p))
    for name, (t, b, p) in list(key_value_cases().items()) + list(null_cases().items()):
        out.append((name, t, b, p))
    for s in BUCKET_SIZES:
        b, p = bucket_case(s)
        out.append((f"bucket_{s}", T_I64, b, p))
    b, p = all_buckets_case()
    out.append(("all_buckets", T_I64, b, p))
    return out


# =============================================================================================================================
# CPU part
# =============================================================================================================================
@pytest.fixture(scope="module")
def H(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("join_hash") / "join_hash_host.so")
    subprocess.check_call(["g++", "-O1", "-x", "c++", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "join_hash_host.cpp")])
    L = ct.CDLL(so)
    for f in ("h_mix64", "h_key_hash_i64", "h_key_hash_bytes"):
        getattr(L, f).restype = ct.c_ulonglong
    L.h_mix64.argtypes = L.h_key_hash_i64.argtypes = [ct.c_ulonglong]
    L.h_key_hash_bytes.argtypes = [ct.c_char_p, ct.c_uint]
    return L


def test_key_hash_restatement_matches_header(H):
    rng = np.random.default_rng(7)
    ints = I64_EDGES + I64_ABSENT + [INT64_MIN | 1, 0x1E3779B97F4A7C15, -0x1E3779B97F4A7C15] + [int(v) for v in rng.integers(INT64_MIN, INT64_MAX, 3000, dtype=np.int64)]
    for v in ints:
        assert H.h_mix64(v & M64) == mix64(v & M64), v
        assert H.h_key_hash_i64(v & M64) == hash_i64(v), v
    vals = np.array(ints, np.int64)
    assert _np_home_i64(vals).tolist() == [home(hash_i64(v)) for v in ints]
    strs = [b"", b"\0", b"\0" * 3, b"\xff" * 2, b"a", b"a\0"]
    for ln in range(258):
        strs.append(rng.integers(0, 256, ln, dtype=np.uint8).tobytes())
        strs.append(bytes([0x80 + (ln % 128)]) * ln)
    for s in strs:
        assert H.h_key_hash_bytes(s, len(s)) == hash_bytes(s), s
    for ln in (0, 1, 8, 33):
        mat = rng.integers(0, 256, (50, ln), dtype=np.uint8)
        assert _np_home_bytes(mat).tolist() == [home(hash_bytes(r.tobytes())) for r in mat]


def test_colliding_key_sets_collide_as_designed():
    for build, probe, g in (colliding_i64(), colliding_str()):
        assert len(build) <= CAP // 2  # so the table has CAP slots
        assert {_key_home(k) for k in g["wrap"] + g["wrap_absent"]} == {CAP - 1}
        occ = _table_slots(list(dict.fromkeys(build)))
        assert occ[CAP - 1] and occ[0], "the cluster at slot cap - 1 does not wrap to slot 0"
        for k in g["wrap_absent"]:
            assert k not in build and _walk(occ, CAP - 1) >= len(g["wrap"])  # a miss that walks the whole wrapped cluster
        for a, b in g["pairs"]:
            assert a != b and _key_home(a) == _key_home(b)
        for k in g["pair_absent"]:
            assert k not in build and k in probe
        assert len(g["pairs"]) >= 4
    _, _, gi = colliding_i64()
    for a, b in gi["pairs"]:
        assert (a - b) % (1 << 32) == 0  # equal low 32 bits
    assert any(k < 0 for p in gi["pairs"] for k in p)
    for k in gi["cluster_absent"]:
        assert _key_home(k) in (0, 1, 2) and k not in colliding_i64()[0]
    _, _, gs = colliding_str()
    assert sorted({len(a) for a, _ in gs["pairs"]}) == [1, 2, 3, 7, 16, 17, 31, 64, 129, 256, 257]
    for a, b in gs["pairs"]:
        assert len(a) == len(b) and a[:-1] == b[:-1]
    assert len(gs["len_pairs"]) >= 2
    for a, b in gs["len_pairs"]:
        assert b == a + b"\0" and _key_home(a) == _key_home(b)


def test_string_key_starts_cover_every_offset_mod_16():
    _, b, p = key_value_cases()["str"]
    for keys in (b, p):
        c = scol(keys)
        starts = {int(c.offsets[i]) % 16 for i, k in enumerate(keys) if k}
        assert starts == set(range(16))


def _pairs_via_interpreter(bkeys, pkeys, left_outer):
    L = [(k, i) for i, k in enumerate(pkeys)]
    R = [(k, j) for j, k in enumerate(bkeys)]
    rows = dataset._py_join_pairs(L, 0, R, 0, left_outer, True, 2)
    return np.array([r[0] for r in rows], np.int64), np.array([-1 if r[2] is None else r[2] for r in rows], np.int64)


@pytest.mark.parametrize("left_outer", [False, True])
def test_reference_matches_oracle_and_interpreter(left_outer):
    """The reference against the C join oracle and the interpreter path's join, over the whole small-case matrix."""
    for name, t, bkeys, pkeys in small_key_matrix():
        op, ob = ref_pairs_values(bkeys, pkeys, left_outer)
        bc, pc = _kcol(t, bkeys), _kcol(t, pkeys)
        assert key_values(bc) == [None if k is None else (bool(k) if t == T_BOOL else k) for k in bkeys]
        oop, oob = po.join_pairs(bc, len(bkeys), pc, len(pkeys), left_outer)
        assert np.array_equal(op, oop) and np.array_equal(ob, oob), name
        iop, iob = _pairs_via_interpreter(bkeys, pkeys, left_outer)
        assert np.array_equal(op, iop) and np.array_equal(ob, iob), name
        if t == T_I64 and None not in bkeys and None not in pkeys:
            nop, nob = ref_pairs_np(np.array(bkeys, np.int64), np.array(pkeys, np.int64), left_outer)
            assert np.array_equal(op, nop) and np.array_equal(ob, nob), name


def test_numpy_reference_matches_dict_reference():
    rng = np.random.default_rng(8)
    for nb, npr, nk in [(0, 5, 3), (5, 0, 3), (1, 1, 1), (300, 500, 40), (2000, 3000, 5000)]:
        b, p = rng.integers(-nk, nk, nb), rng.integers(-nk, nk + 5, npr)
        for lo in (False, True):
            op, ob = ref_pairs_values(b.tolist(), p.tolist(), lo)
            nop, nob = ref_pairs_np(b, p, lo)
            assert np.array_equal(op, nop) and np.array_equal(ob, nob)


def test_type_tags_keep_bool_and_int_apart():
    op, ob = ref_pairs_values([1, True, 0, False, None], [True, 1, False, 0, None], False)
    assert list(zip(op.tolist(), ob.tolist())) == [(0, 1), (1, 0), (2, 3), (3, 2), (4, 4)]


# =============================================================================================================================
# GPU part: backend.Join / probe
# =============================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", ["colliding_i64", "colliding_str"])
def test_gpu_colliding_keys(gpu, case, mode):
    bkeys, pkeys, g = colliding_i64() if case == "colliding_i64" else colliding_str()
    t = T_I64 if case == "colliding_i64" else T_STR
    build, probe = with_payloads(_kcol(t, bkeys), b"b", 1), with_payloads(_kcol(t, pkeys), b"p", 2)
    op, ob, info = check_join(build, 1, probe, 2, mode)
    # every key of a colliding pair found its own rows and only those
    matched = {}
    for i, j in zip(op.tolist(), ob.tolist()):
        if j >= 0:
            matched.setdefault(pkeys[i], set()).add(bkeys[j])
    for a, b in g["pairs"]:
        assert matched[a] == {a} and matched[b] == {b}
    assert not any(k in matched for k in g["wrap_absent"] + g["pair_absent"])
    assert info["n_rows"] == len(bkeys)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", ["i64", "bool", "bool_no_none", "str", "str_empty_vs_none"])
def test_gpu_key_values(gpu, case, mode):
    t, bkeys, pkeys = key_value_cases()[case]
    build, probe = with_payloads(_kcol(t, bkeys), b"b"), with_payloads(_kcol(t, pkeys), b"p", 2)
    op, ob, info = check_join(build, 0, probe, 2, mode)
    assert info["n_null_rows"] == sum(k is None for k in bkeys)
    if case == "str_empty_vs_none":  # "" matches "" only, None matches None only
        assert list(zip(op.tolist(), ob.tolist()))[:6] == [(0, 2), (1, 0), (1, 1), (2, 3), (3, 2), (4, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", ["both_0", "both_1", "both_33", "both_2049", "build_only", "probe_only", "all_null_build", "str_both"])
def test_gpu_null_keys(gpu, case, mode):
    t, bkeys, pkeys = null_cases()[case]
    build, probe = with_payloads(_kcol(t, bkeys), b"b", 2), with_payloads(_kcol(t, pkeys), b"p")
    _, _, info = check_join(build, 2, probe, 0, mode)
    assert info["n_null_rows"] == sum(k is None for k in bkeys)
    largest = max(Counter(_tag(k) for k in bkeys).values())  # the null bucket is one of the groups
    assert info["kernel_launches"] == (8 if largest > 32 else 6)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("size", BUCKET_SIZES)
def test_gpu_bucket_sizes(gpu, size, mode):
    """A bucket of `size` rows spread over the build side, probed from warps that mix wide rows, narrow rows and misses. Buckets
    above 32 rows are ordered by join_order_big (8 launches for the build), smaller ones by join_order_small alone (6)."""
    bkeys, pkeys = bucket_case(size)
    build, probe = with_payloads(icol(bkeys), b"b"), with_payloads(icol(pkeys), b"p", 1)
    op, ob, info = check_join(build, 0, probe, 1, mode)
    assert info["kernel_launches"] == (8 if size > 32 else 6)
    rows7 = [j for j, k in enumerate(bkeys) if k == 7]
    assert len(rows7) == size and (size < 31 or rows7[-1] - rows7[0] > len(bkeys) // 2)  # spread over the build side
    for i in np.flatnonzero(np.array(pkeys) == 7).tolist():
        assert ob[op == i].tolist() == rows7


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_gpu_all_bucket_sizes_in_one_table(gpu, mode):
    bkeys, pkeys = all_buckets_case()
    build, probe = with_payloads(icol(bkeys), b"b", 2), with_payloads(icol(pkeys), b"p")
    op, ob, info = check_join(build, 2, probe, 0, mode)
    assert info["kernel_launches"] == 8
    for k, s in enumerate(BUCKET_SIZES):  # every bucket's build rows, in build-row order
        rows = [j for j, v in enumerate(bkeys) if v == k]
        assert len(rows) == s
        i = pkeys.index(k)
        assert ob[op == i].tolist() == rows


F64_EDGE_BITS = [0x0000000000000000, 0x8000000000000000, 0x7FF8000000000001, 0x7FF0000000000001, 0xFFF8000000000ABC, 0x7FF4000000000000,
                 0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001, 0x3FF8000000000000, 0xFFFFFFFFFFFFFFFF]


def _payload_side(rng, keys, key_type, key_pos, tag):
    """The key at key_pos among i64, bool, str and f64 payloads and the Option variant of each (None in about a third of the rows)."""
    n = len(keys)
    some = rng.random(n) < 0.35

    def opt(vals):
        return [None if s else v for v, s in zip(vals, some.tolist())]
    i64 = [INT64_MIN, INT64_MAX, 0, -1, 1 << 32] + rng.integers(INT64_MIN, INT64_MAX, max(n - 5, 0), dtype=np.int64).tolist()
    i64 = i64[:n]
    bools = (rng.random(n) < 0.5).tolist()
    strs = [(b"%s%d\xff\0" % (tag, i)) * int(i % 4) for i in range(n)]
    fbits = [F64_EDGE_BITS[i % len(F64_EDGE_BITS)] for i in range(n)]
    cols = [icol(i64), icol(bools, T_BOOL), scol(strs), fcol_bits(fbits),
            icol(opt(i64)), icol(opt(bools), T_BOOL), scol(opt(strs)), fcol_bits(fbits, (~some).tolist())]
    assert all(c.valid is not None for c in cols[4:])
    cols.insert(key_pos, _kcol(key_type, keys))
    return cols


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n_out", [64, 65, 95])
@pytest.mark.parametrize("key_pos", [0, 4, 8])
def test_gpu_payloads_both_sides(gpu, key_pos, n_out, mode):
    """Every payload type and its Option variant on both sides, the key first, in the middle or last on each side; n_out % 32 of 0, 1
    and 31, so the last validity word is checked."""
    rng = np.random.default_rng(14 + key_pos + n_out)
    kt = T_STR if key_pos == 4 else T_I64
    mk = (lambda v: b"key%d" % v) if kt == T_STR else (lambda v: v * 7919 - 40)
    n_build = 100
    bkeys = [mk(v) for v in rng.permutation(n_build).tolist()]
    n_match = n_out if mode != "left" else n_out - 13
    pkeys = [mk(int(v)) for v in rng.integers(0, n_build, n_match)] + [mk(n_build + i) for i in range(13)]
    pkeys = _spread(rng, pkeys)
    build = _payload_side(rng, bkeys, kt, key_pos, b"b")
    probe = _payload_side(rng, pkeys, kt, 8 - key_pos, b"p")
    op, _, _ = check_join(build, key_pos, probe, 8 - key_pos, mode)
    assert len(op) == n_out


def _size_table(rng):
    keys = _spread(rng, [k for k in range(120) for _ in range(1 + k % 40)])
    return with_payloads(icol(keys), b"b", 1)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n_probe", [0, 1, 255, 256, 257, 2047, 2048, 2049])
def test_gpu_probe_block_sizes(gpu, n_probe, mode):
    rng = np.random.default_rng(15 + n_probe)
    build = _size_table(rng)
    probe = with_payloads(icol(rng.integers(-5, 130, n_probe).tolist()), b"p")
    op, _, _ = check_join(build, 1, probe, 0, mode)
    if n_probe == 0:
        assert len(op) == 0


def _big_str(rng, n, tag):
    """n strings of 0-12 bytes built with numpy (row i's bytes depend on i and the tag)."""
    lens = (np.arange(n) * 7 + len(tag)) % 13
    off = np.zeros(n + 1, np.uint32)
    np.cumsum(lens, out=off[1:])
    data = rng.integers(0, 256, int(off[-1]), dtype=np.uint8)
    return Column(T_STR, data, off)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_gpu_probe_of_2_1m_rows_with_over_2_21_output_rows(gpu, mode):
    """2,100,000 probe rows (count scan over more than 2^21 entries) and more than 2^21 output rows with string columns on both
    sides (string-length scans over more than 2^21 entries)."""
    rng = np.random.default_rng(16)
    n_build, n_probe = 5000, 2_100_000
    bkeys = rng.integers(0, 4000, n_build)
    pkeys = rng.integers(0, 4200, n_probe)
    build = [Column(T_I64, bkeys), Column(T_I64, np.arange(n_build, dtype=np.int64)), _big_str(rng, n_build, "b")]
    probe = [_big_str(rng, n_probe, "pp"), Column(T_I64, pkeys), Column(T_I64, rng.integers(INT64_MIN, INT64_MAX, n_probe, dtype=np.int64))]
    pairs = ref_pairs_np(bkeys, pkeys, mode == "left")
    op, _, _ = check_join(build, 0, probe, 1, mode, pairs)
    assert len(op) > (1 << 21)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_gpu_build_of_2_20_rows(gpu, mode):
    """2^20 build rows: the bench's table capacity of 2^21, whose group scan has 1025 block sums."""
    rng = np.random.default_rng(17)
    n_build, n_probe = 1 << 20, 300_000
    bkeys = rng.integers(-(1 << 40), 1 << 40, 700_000)[rng.integers(0, 700_000, n_build)]
    pkeys = np.concatenate([bkeys[rng.integers(0, n_build, n_probe - 50_000)], rng.integers(-(1 << 40), 1 << 40, 50_000)])
    rng.shuffle(pkeys)
    build = [Column(T_I64, np.arange(n_build, dtype=np.int64)), Column(T_I64, bkeys)]
    probe = [Column(T_I64, pkeys), _big_str(rng, n_probe, "p")]
    pairs = ref_pairs_np(bkeys, pkeys, mode == "left")
    _, _, info = check_join(build, 1, probe, 0, mode, pairs)
    assert info["n_rows"] == n_build


@pytest.mark.gpu
def test_gpu_table_reuse(gpu):
    """One table probed by several blocks, the same block probed twice, and two live tables probed alternately on one device."""
    rng = np.random.default_rng(18)
    b1 = with_payloads(icol(_spread(rng, [k for k in range(200) for _ in range(1 + k % 35)])), b"x")
    b2 = with_payloads(scol(_spread(rng, [b"s%d" % (k % 90) for k in range(400)])), b"y", 2)
    bb1, bb2 = backend.Block.upload(0, b1, nrows(b1)), backend.Block.upload(0, b2, nrows(b2))
    j1, j2 = backend.Join(bb1, [c.type for c in b1], 0), backend.Join(bb2, [c.type for c in b2], 2)
    try:
        blocks = [with_payloads(icol(rng.integers(-3, 210, n).tolist()), b"p", 1) for n in (300, 1000, 37)]
        for p in blocks + [blocks[0]]:
            for mode in MODES:
                check_probe(j1, b1, 0, p, 1, mode)
        sblocks = [with_payloads(scol([b"s%d" % v for v in rng.integers(0, 100, n).tolist()]), b"q") for n in (50, 700)]
        for p, s in [(blocks[0], sblocks[0]), (blocks[1], sblocks[1]), (blocks[2], sblocks[0])]:
            check_probe(j1, b1, 0, p, 1, "left")
            check_probe(j2, b2, 2, s, 0, "left")
            check_probe(j2, b2, 2, s, 0, "build_first")
    finally:
        j1.free()
        j2.free()
        bb1.free()
        bb2.free()


@pytest.mark.gpu
def test_gpu_output_column_limit(gpu):
    """TPLX_MAX_COLS output columns are accepted; one more raises GpuBackendError."""
    rng = np.random.default_rng(19)
    n_probe_cols = backend.MAX_COLS // 2
    n_build_cols = backend.MAX_COLS - n_probe_cols + 1
    bkeys = _spread(rng, list(range(40)) * 2)
    pkeys = rng.integers(-2, 45, 70).tolist()

    def side(keys, n_cols, tag):
        cols = [icol(keys)]
        for c in range(1, n_cols):
            cols.append(scol([b"%s%d.%d" % (tag, c, i) for i in range(len(keys))]) if c % 3 == 0 else icol([c * 1000 + i for i in range(len(keys))]))
        return cols
    build, probe = side(bkeys, n_build_cols, b"b"), side(pkeys, n_probe_cols, b"p")
    for mode in MODES:
        check_join(build, 0, probe, 0, mode)
    wide = build + [icol(list(range(len(bkeys))))]
    bb = backend.Block.upload(0, wide, len(bkeys))
    pb = backend.Block.upload(0, probe, len(pkeys))
    j = backend.Join(bb, [c.type for c in wide], 0)
    try:
        for mode in MODES:
            with pytest.raises(backend.GpuBackendError):
                j.probe(pb, [c.type for c in probe], 0, left_outer=mode == "left", build_first=mode == "build_first")
    finally:
        j.free()
        pb.free()
        bb.free()


# ---- Context: join / leftJoin over several probe blocks, with fallback rows and None keys ------------------------------------
def _nested_loop_join(L, li, R, ri, left_outer, build_right):
    """The join over the original Python rows by a nested loop: keys match when both are None, or have one type and are equal."""
    def match(a, b):
        return (a is None and b is None) or (a is not None and b is not None and type(a) is type(b) and a == b)

    def row(lr, rr):
        rr = rr if rr is not None else (None,) * len(R[0])
        return tuple(v for i, v in enumerate(lr) if i != li) + (lr[li],) + tuple(v for i, v in enumerate(rr) if i != ri)
    out = []
    if build_right:
        for lr in L:
            ms = [rr for rr in R if match(lr[li], rr[ri])]
            out += [row(lr, rr) for rr in ms]
            if left_outer and not ms:
                out.append(row(lr, None))
    else:
        for rr in R:
            out += [row(lr, rr) for lr in L if match(lr[li], rr[ri])]
    return out


def _context_rows(n_left, n_right):
    rng = np.random.default_rng(20)
    L = [(int(k), "l%d" % i) for i, k in enumerate(rng.integers(0, 150, n_left))]
    R = [(int(k), float(i)) for i, k in enumerate(rng.integers(0, 200, n_right))]
    for i in range(0, n_left, 97):
        L[i] = (None, "ln%d" % i)       # None keys on both sides: they match each other
    for i in range(5, n_right, 41):
        R[i] = (None, -float(i))
    L[17] = ("seventeen", "odd")        # key of another type: a fallback row ...
    R[11] = ("seventeen", 2.5)          # ... that matches a fallback row of the other side
    L[n_left - 2] = (5, 123)            # payload of another type
    R[3] = (100000, "only")             # a build-side fallback row (payload of another type) ...
    L[40] = (100000, "l40")             # ... which is this left row's only match
    L[n_left // 2] = (100000, "again")
    R[n_right - 1] = (1 << 70, 1.0)     # key beyond 64 bits
    L[60] = (1 << 70, "big")
    return L, R


@pytest.mark.gpu
@pytest.mark.parametrize("kind,build_right", [("join", True), ("join", False), ("leftJoin", True)])
def test_context_join_with_fallback_rows_and_none_keys(gpu, kind, build_right):
    import tuplex_b200 as tuplex
    L, R = _context_rows(2500, 300) if build_right else _context_rows(300, 2500)
    c = tuplex.Context({"tuplex.gpu.blockRows": 777})
    dl, dr = c.parallelize(L, columns=["k", "v"]), c.parallelize(R, columns=["k", "w"])
    ds = dl.leftJoin(dr, "k", "k") if kind == "leftJoin" else dl.join(dr, "k", "k")
    assert ds._join.build_right() is build_right
    got = ds.collect()
    exp = _nested_loop_join(L, 0, R, 0, kind == "leftJoin", build_right)
    assert got == exp
    assert dataset._py_join_pairs(L, 0, R, 0, kind == "leftJoin", build_right, 2) == exp
    if kind == "leftJoin":
        assert ("l40", 100000, "only") in got and ("l40", 100000, None) not in got
