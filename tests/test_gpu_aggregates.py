"""aggregate / aggregateByKey on the device against exact references computed here from the inputs.

The references are plain Python or numpy over the generated rows: functools.reduce of the user's own UDFs, Python integers
reduced mod 2^64 (i64 sums wrap, tplx_ir.h), math.fsum, and np.minimum.at / np.add.at per group. None of them comes from the
C oracle, which restates the kernels' accumulator code and so shares any mistake in it.

f64 sums are made exact: every summed value is k / 64 with |k| < 2^20 and there are fewer than 2^26 rows, so every partial
sum in any order is representable. The K3 tree, the K4 atomics and the table merge then all have to give the exact sum, and
a dropped or duplicated row changes it whatever the order.

K3 = stage_agg_kernel / specialised agg kernel + agg_finalize_kernel (tile of 4096 rows, finalize folds tile += 1024);
K4 = stage_hash_kernel (shared-memory pre-aggregation buckets, then the table) + hash_emit.
The last section runs without a GPU: the front end's lowering of min/max and the host folds against CPython."""
import functools
import math

import numpy as np
import pytest

import tuplex_b200
from tuplex_b200 import backend, dataset, frontend, ir
from tuplex_b200.backend import Block, Column
from tuplex_b200.ir import C, T_BOOL, T_F64, T_I64, T_STR

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
MASK = (1 << 64) - 1
INF = float("inf")
SUBNORMAL = 5e-324
TILE = 4096  # K3 rows per tile (R = 16 x 256 threads)
KINDS6 = [C["TPLX_ACC_MIN_I64"], C["TPLX_ACC_MAX_I64"], C["TPLX_ACC_SUM_I64"],
          C["TPLX_ACC_MIN_F64"], C["TPLX_ACC_MAX_F64"], C["TPLX_ACC_SUM_F64"]]
F64_KINDS = {C["TPLX_ACC_MIN_F64"], C["TPLX_ACC_MAX_F64"], C["TPLX_ACC_SUM_F64"]}


# one accumulator of every kind: i64 min / max / sum over a, b, c; f64 min / max / sum over d, e, f
def AGG6(a, x):
    return (min(a[0], x["a"]), max(a[1], x["b"]), a[2] + x["c"], min(a[3], x["d"]), max(a[4], x["e"]), a[5] + x["f"])


def COMB6(a, b):
    return (min(a[0], b[0]), max(a[1], b[1]), a[2] + b[2], min(a[3], b[3]), max(a[4], b[4]), a[5] + b[5])


# no component is an identity; the f64 min starts from an int
INIT6 = (1 << 50, -(1 << 50), 12345, 1 << 30, -2.0 ** 30, 0.25)
IDENT6 = (I64_MAX, I64_MIN, 0, INF, -INF, 0.0)
NAMES6 = ["a", "b", "c", "d", "e", "f"]
TYPES6 = [T_I64, T_I64, T_I64, T_F64, T_F64, T_F64]


def wrap(v: int) -> int:
    v &= MASK
    return v - (1 << 64) if v >= 1 << 63 else v


def bits6(vals) -> list:
    """Accumulator values (Python numbers) -> the 64-bit patterns the device returns."""
    return [ir.f64_bits(float(v)) if k in F64_KINDS else wrap(int(v)) & MASK for k, v in zip(KINDS6, vals)]


def finish6(bucket):
    """LocalBackend applyCombinePerGroup on a bucket that itself started from init: combine(init, combine(init, bucket))."""
    v = COMB6(INIT6, COMB6(INIT6, bucket))
    return v[:2] + (wrap(v[2]),) + v[3:]


def values6(rng, n):
    """Random accumulator inputs: i64 min/max in +-2^40, i64 sum over the whole range (wraps), f64 as k / 64."""
    return {"a": rng.integers(-(1 << 40), 1 << 40, n), "b": rng.integers(-(1 << 40), 1 << 40, n),
            "c": rng.integers(I64_MIN, I64_MAX, n, endpoint=True),
            "d": rng.integers(-(1 << 19), 1 << 19, n) / 64.0, "e": rng.integers(-(1 << 19), 1 << 19, n) / 64.0,
            "f": rng.integers(-(1 << 20) + 1, 1 << 20, n) / 64.0}


def rows_of(cols: dict, idx) -> list:
    """Rows as dicts of Python scalars (what the user's UDF sees)."""
    lists = {k: v.tolist() if isinstance(v, np.ndarray) else list(v) for k, v in cols.items()}
    return [{k: lists[k][i] for k in lists} for i in idx]


def ccol(v, t) -> Column:
    if t in (T_STR, T_BOOL):
        return Column.from_values(list(v), t)
    return Column(t, np.ascontiguousarray(v, dtype=np.float64 if t == T_F64 else np.int64))


@pytest.fixture(params=[0, 2], ids=["interpreted", "specialised"])
def jit_mode(request, monkeypatch):
    """TPLX_JIT=0: interpreting kernels only; TPLX_JIT=2 + TPLX_JIT_SYNC=1: every stage specialised at its first block."""
    monkeypatch.setenv("TPLX_JIT", str(request.param))
    if request.param == 2:
        monkeypatch.setenv("TPLX_JIT_SYNC", "1")
    else:
        monkeypatch.delenv("TPLX_JIT_SYNC", raising=False)
    return request.param


# =============================================================================================================================
# K3: aggregate
# =============================================================================================================================
def k3_program():
    sc = frontend.StageCompiler(TYPES6 + [T_I64], NAMES6 + ["m"])
    sc.add_filter(lambda x: x["m"] != 3, 100001)
    return sc.finish_aggregate(AGG6, COMB6, INIT6, 100002)


def k3_placements(n):
    """Row 0, the last row of tile 0, the first row of tile 1, the last row of the last full tile, the last row."""
    last_full = (n // TILE) * TILE - 1
    return sorted({p for p in (0, TILE - 1, TILE, last_full, n - 1) if 0 <= p < n})


# extremes per variant: A = identities of min/max and infinities; B = data equal to the identities, subnormal results,
# an extra exact f64 term
EXTREME = {"A": (I64_MIN, I64_MAX, I64_MAX, -INF, INF, INF),
           "B": (-1, 1, I64_MIN, SUBNORMAL, -SUBNORMAL, 2.0 ** 40 + 1 / 64)}


def k3_data(rng, n, variant):
    v = values6(rng, n)
    if variant == "B":
        v["a"] = np.full(n, I64_MAX, np.int64)  # min over values equal to the identity
        v["b"] = np.full(n, I64_MIN, np.int64)
        v["d"] = rng.integers(1, 1 << 20, n) / 64.0
        v["e"] = -rng.integers(1, 1 << 20, n) / 64.0
    v["m"] = rng.integers(0, 8, n)
    return v


def k3_reference(v, keep):
    """init (+) fold of the kept rows; i64 sum as a Python integer mod 2^64, f64 sum by fsum (exact here)."""
    if not keep.any():
        return INIT6[:2] + (wrap(INIT6[2]),) + INIT6[3:]
    return (min(INIT6[0], int(v["a"][keep].min())), max(INIT6[1], int(v["b"][keep].max())),
            wrap(INIT6[2] + sum(v["c"][keep].tolist())),
            min(INIT6[3], float(v["d"][keep].min())), max(INIT6[4], float(v["e"][keep].max())),
            INIT6[5] + math.fsum(v["f"][keep].tolist()))


def run_k3(st, v, n):
    res = st.run_host(0, [ccol(v[k], t) for k, t in zip(NAMES6 + ["m"], TYPES6 + [T_I64])], n)
    return res.aggregate_bits(), res.info


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 31, 4095, 4096, 4097, 1_048_577, 4 * 1024 * 1024 + 4097])
def test_k3_min_max_sum_all_kinds(gpu, jit_mode, n):
    """Six accumulators, one per kind, at tile edges and past 1024 tiles (the finalize kernel's second pass); the extreme row
    sits at each of the rows a reduction can lose; interpreted and specialised kernels."""
    prog = k3_program()
    assert [a.kind for a in prog.accs] == KINDS6
    st = backend.Stage(prog)
    rng = np.random.default_rng(1000 + n)
    for variant in ("A", "B"):
        v = k3_data(rng, n, variant)
        places = k3_placements(n)
        v["m"][places] = 3  # filtered in the base: each placement below adds exactly one row
        keep = v["m"] != 3
        base = k3_reference(v, keep)
        if n <= 2 * TILE:  # the numpy reference is the user's UDF folded in CPython
            red = functools.reduce(AGG6, rows_of(v, np.flatnonzero(keep)), INIT6)
            assert bits6(red[:2] + (wrap(red[2]),) + red[3:]) == bits6(base)
        bits, info = run_k3(st, v, n)
        assert bits == bits6(base), f"n={n} {variant} without the extreme row"
        assert (int(info.specialised_launches) > 0) == (jit_mode == 2 and n > 0)
        for p in places:
            old = {k: v[k][p] for k in NAMES6}
            for k, x in zip(NAMES6, EXTREME[variant]):
                v[k][p] = x
            v["m"][p] = 0
            want = COMB6(base, tuple(EXTREME[variant]))
            want = want[:2] + (wrap(want[2]),) + want[3:]
            assert all(bits6(want)[i] != bits6(base)[i] for i in range(6)), "the extreme row must change every accumulator"
            bits, info = run_k3(st, v, n)
            assert bits == bits6(want), f"n={n} {variant}: extreme row at {p}"
            for k in NAMES6:
                v[k][p] = old[k]
            v["m"][p] = 3


@pytest.mark.gpu
def test_k3_filter_removes_every_row_gives_init(gpu, jit_mode):
    st = backend.Stage(k3_program())
    rng = np.random.default_rng(7)
    for n in (0, 1, 5000, TILE * 3 + 1):
        v = k3_data(rng, n, "A")
        v["m"][:] = 3
        bits, info = run_k3(st, v, n)
        assert bits == bits6(INIT6[:2] + (wrap(INIT6[2]),) + INIT6[3:]), f"n={n}"
        assert int(info.n_exceptions) == 0


@pytest.mark.gpu
def test_k3_nan_rows_are_ignored_by_min_max(gpu, jit_mode):
    """CPython's answer for min(x, a) depends on where a NaN sits; the device ignores NaN rows in every spelling (DESIGN §4)."""
    n = 3 * TILE + 5
    rng = np.random.default_rng(8)
    d = rng.integers(-(1 << 19), 1 << 19, n) / 64.0
    d[[0, TILE, n - 1]] = np.nan
    sc = frontend.StageCompiler([T_F64], ["d"])
    prog = sc.finish_aggregate(lambda a, x: (min(x["d"], a[0]), max(a[1], x["d"]), min(a[2], x["d"])),
                               lambda a, b: (min(a[0], b[0]), max(a[1], b[1]), min(a[2], b[2])), (INF, -INF, INF), 100001)
    res = backend.Stage(prog).run_host(0, [ccol(d, T_F64)], n)
    lo, hi = float(np.nanmin(d)), float(np.nanmax(d))
    assert res.aggregate_bits() == [ir.f64_bits(lo), ir.f64_bits(hi), ir.f64_bits(lo)]


@pytest.mark.gpu
def test_k3_exception_rows_past_the_first_capacity_estimate(gpu, jit_mode):
    """~10 % of the rows raise ValueError in int(): more than the first exception buffer (max(4096, n/64)) holds, so run_agg
    takes its second attempt. Every raising row comes back, numbered in row order, and the aggregate covers the others."""
    n = 200_000
    rng = np.random.default_rng(9)
    num = rng.integers(-(1 << 40), 1 << 40, n)
    bad = rng.random(n) < 0.1
    num[np.flatnonzero(bad)[:1]] = -(1 << 50)  # the smallest value sits in a raising row: it must not count
    s = ["x%d" % q if b else str(q) for q, b in zip(num.tolist(), bad.tolist())]
    f = rng.integers(-(1 << 20) + 1, 1 << 20, n) / 64.0
    sc = frontend.StageCompiler([T_STR, T_F64], ["s", "f"])
    sc.add_with_column("v", lambda x: int(x["s"]), 100001)
    prog = sc.finish_aggregate(lambda a, x: (min(a[0], x["v"]), max(a[1], x["v"]), a[2] + x["v"], min(a[3], x["f"]), max(a[4], x["f"]), a[5] + x["f"]),
                               COMB6, INIT6, 100002)
    res = backend.Stage(prog).run_host(0, [ccol(s, T_STR), ccol(f, T_F64)], n)
    exc = res.exceptions()
    want_rows = np.flatnonzero(bad)
    assert int(res.info.n_exceptions) == len(want_rows) > 4096 + n // 64
    assert np.array_equal(exc["row"], want_rows)
    assert np.array_equal(exc["row_no"], np.arange(len(want_rows)))
    assert set(exc["op_id"].tolist()) == {100001} and set(exc["code"].tolist()) == {C["TPLX_EC_VALUEERROR"]}
    ok = ~bad
    want = (min(INIT6[0], int(num[ok].min())), max(INIT6[1], int(num[ok].max())), wrap(INIT6[2] + sum(num[ok].tolist())),
            min(INIT6[3], float(f[ok].min())), max(INIT6[4], float(f[ok].max())), INIT6[5] + math.fsum(f[ok].tolist()))
    assert res.aggregate_bits() == bits6(want)


# =============================================================================================================================
# K4: aggregateByKey
# =============================================================================================================================
def group_reference(keys: list, rows: list) -> dict:
    """key tuple -> bucket (the user's aggregate UDF folded from the identities, as the device's bucket is)."""
    out = {}
    for k, r in zip(keys, rows):
        out[k] = AGG6(out.get(k, IDENT6), r)
    return out


def fetch_groups(res, nk: int) -> dict:
    cols = res.columns()
    keys = list(zip(*[c.to_values() for c in cols[:nk]]))
    accs = [[ir.f64_bits(x) if k in F64_KINDS else x & MASK for x in cols[nk + i].data.tolist()] for i, k in enumerate(KINDS6)]
    assert len(set(keys)) == len(keys), "a key was emitted twice"
    return {k: [accs[i][j] for i in range(6)] for j, k in enumerate(keys)}


def hash_program(key_names, key_types):
    sc = frontend.StageCompiler(TYPES6 + list(key_types), NAMES6 + list(key_names))
    prog = sc.finish_hash(list(key_names), AGG6, COMB6, INIT6, 100001)
    assert [a.kind for a in prog.accs] == KINDS6
    return prog


def with_edges(rng, v, n):
    """Sprinkle the min/max identities and infinities over ~0.2 % of the rows."""
    for k, x in (("a", I64_MIN), ("b", I64_MAX), ("d", -INF), ("e", INF), ("a", I64_MAX), ("b", I64_MIN)):
        v[k][rng.integers(0, n, max(1, n // 3000))] = x
    return v


STRS = ["", "a", "ä", "日本語", "aä", "zillow, boston", "x" * 40, "Ünïcödé ✓"]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["i64_str_bool", "str_str"])
def test_k4_all_kinds_multi_column_keys_two_blocks(gpu, layout):
    """Mixed key blobs (i64 8 bytes, str len + bytes, bool), empty and non-ASCII strings, two blocks into one table."""
    if layout == "i64_str_bool":
        names, types = ["k1", "k2", "k3"], [T_I64, T_STR, T_BOOL]
    else:
        names, types = ["k2", "k4"], [T_STR, T_STR]
    st = backend.Stage(hash_program(names, types))
    rng = np.random.default_rng(11 if layout == "i64_str_bool" else 12)
    k1_pool = np.array([I64_MIN, I64_MAX, -1, 0, 1, 1 << 40] + list(range(2, 200)), np.int64)
    all_keys, all_rows = [], []
    for blk in range(2):
        n = 60_000 + 777 * blk
        v = with_edges(rng, values6(rng, n), n)
        kv = {"k1": k1_pool[rng.integers(0, len(k1_pool), n)].tolist(), "k2": [STRS[i] for i in rng.integers(0, len(STRS), n)],
              "k3": [bool(i) for i in rng.integers(0, 2, n)], "k4": [STRS[i] + str(j) if j < 3 else STRS[i] for i, j in
                                                                 zip(rng.integers(0, len(STRS), n), rng.integers(0, 6, n))]}
        st.run_host(0, [ccol(v[k], t) for k, t in zip(NAMES6, TYPES6)] + [ccol(kv[k], t) for k, t in zip(names, types)], n).info
        all_keys += list(zip(*[kv[k] for k in names]))
        all_rows += rows_of(v, range(n))
    got = fetch_groups(st.hash_finish(0), len(names))
    want = {k: bits6(finish6(b)) for k, b in group_reference(all_keys, all_rows).items()}
    assert len(want) > 50
    assert got.keys() == want.keys()
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, f"{len(bad)} of {len(want)} groups differ, e.g. {bad[0]}: {got[bad[0]]} != {want[bad[0]]}"
    # the finish rule written out for the sum with init != 0: init + (init + bucket)
    k0 = next(iter(want))
    bucket = group_reference(all_keys, all_rows)[k0]
    assert got[k0][2] == wrap(INIT6[2] + (INIT6[2] + bucket[2])) & MASK
    assert got[k0][5] == ir.f64_bits(INIT6[5] + (INIT6[5] + bucket[5]))


def numpy_groups(keys, v):
    """Per-group buckets with numpy (ufunc.at): sorted unique keys and six arrays. i64 sums modulo 2^64 in uint64."""
    uk, inv = np.unique(keys, return_inverse=True)
    g = len(uk)
    out = [np.full(g, I64_MAX, np.int64), np.full(g, I64_MIN, np.int64), np.zeros(g, np.uint64),
           np.full(g, INF), np.full(g, -INF), np.zeros(g)]
    np.minimum.at(out[0], inv, v["a"])
    np.maximum.at(out[1], inv, v["b"])
    np.add.at(out[2], inv, v["c"].astype(np.int64).view(np.uint64))
    np.minimum.at(out[3], inv, v["d"])
    np.maximum.at(out[4], inv, v["e"])
    np.add.at(out[5], inv, v["f"])  # every partial sum exact (k / 64 data)
    return uk, out


def numpy_finish_bits(out):
    """combine(init, combine(init, bucket)) per group, as bit patterns."""
    a = np.minimum(out[0], INIT6[0])
    b = np.maximum(out[1], INIT6[1])
    c = out[2] + np.uint64(2 * INIT6[2])
    d = np.minimum(out[3], float(INIT6[3]))
    e = np.maximum(out[4], INIT6[4])
    f = INIT6[5] + (INIT6[5] + out[5])
    return [a.view(np.uint64), b.view(np.uint64), c, d.view(np.uint64), e.view(np.uint64), f.view(np.uint64)]


def assert_table_equals(res, uk, out):
    cols = res.columns()
    order = np.argsort(cols[0].data, kind="stable")
    assert np.array_equal(cols[0].data[order], uk), f"{len(cols[0].data)} keys emitted, {len(uk)} expected"
    want = numpy_finish_bits(out)
    for i in range(6):
        got = cols[1 + i].data[order].view(np.uint64)
        assert np.array_equal(got, want[i]), f"accumulator {i}: {int((got != want[i]).sum())} of {len(uk)} groups differ"


@pytest.mark.gpu
def test_k4_bucket_switch_off_mid_block(gpu):
    """Every tile starts with 16 hot keys, the rest are distinct keys: each CTA's buckets fill, then miss until the
    bucket-disable rule fires mid-block; the buckets' partials must still reach the table at the end."""
    n = 5_000_000
    tile = 1024  # K4 rows per tile (R = 4 x 256 threads)
    r = np.arange(n, dtype=np.int64)
    hot = (r % tile < 64) & (r < 512 * tile)
    keys = np.where(hot, r % 16, 1000 + r)
    rng = np.random.default_rng(13)
    v = values6(rng, n)
    st = backend.Stage(hash_program(["k"], [T_I64]))
    st.run_host(0, [ccol(v[k], t) for k, t in zip(NAMES6, TYPES6)] + [ccol(keys, T_I64)], n).info
    uk, out = numpy_groups(keys, v)
    assert len(uk) == n - int(hot.sum()) + 16
    assert_table_equals(st.hash_finish(0), uk, out)


@pytest.mark.gpu
def test_k4_growth_with_all_kinds(gpu):
    """A reservation far too small: rows that find the table full are retried after hash_rehash, twice over (two blocks)."""
    n = 400_000
    keys = np.arange(n, dtype=np.int64) * 7919 - (1 << 40)
    rng = np.random.default_rng(14)
    st = backend.Stage(hash_program(["k"], [T_I64]))
    st.hash_reserve(0, 1000)
    blocks = [values6(rng, n) for _ in range(2)]
    for v in blocks:
        st.run_host(0, [ccol(v[k], t) for k, t in zip(NAMES6, TYPES6)] + [ccol(keys, T_I64)], n).info
    both = {k: np.concatenate([b[k] for b in blocks]) for k in NAMES6}
    uk, out = numpy_groups(np.concatenate([keys, keys]), both)
    assert_table_equals(st.hash_finish(0), uk, out)


@pytest.mark.gpu
def test_k4_raw_export_and_merge(gpu):
    """The merge half of the multi-GPU exchange on one device: stage A exports raw partials (identities, no init), stage B
    merges them into its own table and finishes; init is applied once, by the finish. Also a merge into an empty stage."""
    n = 120_000
    rng = np.random.default_rng(15)
    v = with_edges(rng, values6(rng, n), n)
    v["e"] = -rng.integers(1, 1 << 20, n) / 64.0  # every f64 max < 0: the raw export must use -inf, not 0, as its identity
    names, types = ["s", "k"], [T_STR, T_I64]
    ks = [STRS[i] for i in rng.integers(0, len(STRS), n)]
    kk = rng.integers(-50, 50, n).tolist()
    prog = hash_program(names, types)
    h = n // 2 + 123

    def cols(lo, hi):
        return [ccol(v[k][lo:hi], t) for k, t in zip(NAMES6, TYPES6)] + [ccol(ks[lo:hi], T_STR), ccol(kk[lo:hi], T_I64)]

    a = backend.Stage(prog)
    a.run_host(0, cols(0, h), h).info
    raw = a.hash_finish(0, raw=True)
    first = group_reference(list(zip(ks[:h], kk[:h])), rows_of(v, range(h)))
    assert fetch_groups(raw, 2) == {k: bits6(b) for k, b in first.items()}, "raw export must be the bucket without init"
    rcols = raw.columns()
    block = Block.upload(0, rcols, int(raw.info.n_out_rows))
    b = backend.Stage(prog)
    b.run_host(0, cols(h, n), n - h).info
    b.hash_merge(block)
    want = {k: bits6(finish6(x)) for k, x in group_reference(list(zip(ks, kk)), rows_of(v, range(n))).items()}
    assert fetch_groups(b.hash_finish(0), 2) == want
    c = backend.Stage(prog)
    c.hash_merge(block)
    assert fetch_groups(c.hash_finish(0), 2) == {k: bits6(finish6(x)) for k, x in first.items()}


# =============================================================================================================================
# K4 exception rows past the buffer (max(4096, n / 32) records)
# =============================================================================================================================
def dirty_ints(rng, n, frac=0.1):
    num = rng.integers(-1000, 1000, n)
    bad = rng.random(n) < frac
    return num, bad, ["%d?" % q if b else str(q) for q, b in zip(num.tolist(), bad.tolist())]


@pytest.mark.gpu
def test_k4_exception_rows_past_the_buffer_stage(gpu):
    n = 300_000
    rng = np.random.default_rng(16)
    num, bad, s = dirty_ints(rng, n)
    keys = rng.integers(0, 97, n)
    sc = frontend.StageCompiler([T_STR, T_I64], ["s", "k"])
    sc.add_with_column("v", lambda x: int(x["s"]), 100001)
    prog = sc.finish_hash(["k"], lambda a, x: a + x["v"], lambda a, b: a + b, 0, 100002)
    st = backend.Stage(prog)
    res = st.run_host(0, [ccol(s, T_STR), ccol(keys, T_I64)], n)
    want_rows = np.flatnonzero(bad)
    got_n = int(res.info.n_exceptions)
    assert got_n == len(want_rows), f"{got_n} exception rows reported, {len(want_rows)} rows raised (buffer {max(4096, n // 32)})"
    exc = res.exceptions()
    assert np.array_equal(exc["row"], want_rows)
    assert np.array_equal(exc["row_no"], np.arange(len(want_rows)))
    assert set(exc["op_id"].tolist()) == {100001}
    fin = st.hash_finish(0)
    got = dict(zip(fin.column(0).data.tolist(), fin.column(1).data.tolist()))
    want = {}
    for k, q in zip(keys[~bad].tolist(), num[~bad].tolist()):
        want[k] = want.get(k, 0) + q
    assert got == want, "normal rows must enter the table once"


@pytest.mark.gpu
@pytest.mark.parametrize("frac", [0.02, 0.1])
def test_k4_exception_rows_survive_table_growth(gpu, frac):
    """A block whose distinct keys outgrow the table: the retry rounds run on a new table, and the block's exception rows
    (below and past the buffer) must still all come back."""
    n = 200_000
    rng = np.random.default_rng(19)
    num, bad, s = dirty_ints(rng, n, frac)
    keys = np.arange(n, dtype=np.int64) * 31
    sc = frontend.StageCompiler([T_STR, T_I64], ["s", "k"])
    sc.add_with_column("v", lambda x: int(x["s"]), 100001)
    st = backend.Stage(sc.finish_hash(["k"], lambda a, x: a + x["v"], lambda a, b: a + b, 0, 100002))
    st.hash_reserve(0, 1000)
    res = st.run_host(0, [ccol(s, T_STR), ccol(keys, T_I64)], n)
    want_rows = np.flatnonzero(bad)
    assert int(res.info.n_exceptions) == len(want_rows), f"{int(res.info.n_exceptions)} exception rows reported, {len(want_rows)} raised"
    assert np.array_equal(res.exceptions()["row"], want_rows)
    fin = st.hash_finish(0)
    order = np.argsort(fin.column(0).data)
    assert np.array_equal(fin.column(0).data[order], keys[~bad])
    assert np.array_equal(fin.column(1).data[order], num[~bad])


def dirty_rows(seed, n):
    rng = np.random.default_rng(seed)
    num, bad, s = dirty_ints(rng, n)
    keys = rng.integers(0, 61, n).tolist()
    return [(k, t, i) for i, (k, t) in enumerate(zip(keys, s))], num, bad


def resolved_v(row):
    """v of a row in CPython: int(s), or the resolver's -(row index) - 1 for rows where int() raises."""
    try:
        return int(row[1])
    except ValueError:
        return -row[2] - 1


@pytest.mark.gpu
def test_k4_exception_rows_past_the_buffer_context(gpu):
    """Three blocks of 100,000 rows, ~10,000 raising rows in each (buffer: 4,096): every raising row is resolved in CPython
    and reaches the groups (aggregateByKey) and the set (unique)."""
    n = 300_000
    rows, num, bad = dirty_rows(17, n)
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 100_000})

    def ds():
        return (ctx.parallelize(rows, columns=["k", "s", "i"]).withColumn("v", lambda x: int(x["s"]))
                .resolve(ValueError, lambda x: -x["i"] - 1))

    want = {}
    for r in rows:
        want[r[0]] = want.get(r[0], 0) + resolved_v(r)
    got = dict(ds().aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["k"]).collect())
    assert got.keys() == want.keys()
    diff = {k: want[k] - got[k] for k in want if got[k] != want[k]}
    assert not diff, f"{len(diff)} of {len(want)} groups differ; sum of the missing row values {sum(diff.values())}"
    got_u = ds().selectColumns(["k", "v"]).unique().collect()
    want_u = {(r[0], resolved_v(r)) for r in rows}
    assert len(got_u) == len(set(got_u)) and set(got_u) == want_u, f"unique: {len(got_u)} rows, {len(want_u)} expected"


@pytest.mark.gpu
def test_context_aggregate_min_max_over_blocks_with_exception_rows(gpu):
    """Context.aggregate with min / max over several blocks: the device partials, the per-block init and the rows resolved in
    CPython give what functools.reduce gives over all rows (min / max are idempotent, so init once per block changes nothing)."""
    n = 250_000
    rows, num, bad = dirty_rows(18, n)
    ctx = tuplex_b200.Context({"tuplex.gpu.blockRows": 60_000})
    agg = lambda a, x: (min(a[0], x["v"]), max(a[1], x["v"]), min(a[2], x["i"] * 0.5), max(a[3], x["k"] - 0.25))  # noqa: E731
    comb = lambda a, b: (min(a[0], b[0]), max(a[1], b[1]), min(a[2], b[2]), max(a[3], b[3]))  # noqa: E731
    init = (10 ** 6, -(10 ** 6), 1e300, -1e300)
    got = (ctx.parallelize(rows, columns=["k", "s", "i"]).withColumn("v", lambda x: int(x["s"]))
           .resolve(ValueError, lambda x: -x["i"] - 1).aggregate(comb, agg, init).collect())
    want = functools.reduce(agg, [{"k": r[0], "i": r[2], "v": resolved_v(r)} for r in rows], init)
    assert want[0] == -int(np.flatnonzero(bad)[-1]) - 1  # the minimum comes from a resolved row
    assert got == [want]


# =============================================================================================================================
# CPU: front-end lowering, oracle and host folds against CPython
# =============================================================================================================================
def lowered(agg, comb, init, endpoint="aggregate"):
    sc = frontend.StageCompiler([T_I64, T_F64, T_I64], ["i", "f", "k"])
    if endpoint == "aggregate":
        prog = sc.finish_aggregate(agg, comb, init, 100001)
    else:
        prog = sc.finish_hash(["k"], agg, comb, init, 100001)
    return [(a.kind, a.init_bits) for a in prog.accs]


@pytest.mark.parametrize("endpoint", ["aggregate", "hash"])
def test_frontend_lowers_every_min_max_spelling(built, endpoint):
    cases = [
        (lambda a, x: min(a, x["i"]), lambda a, b: min(a, b), 0, [(C["TPLX_ACC_MIN_I64"], 0)]),
        (lambda a, x: min(x["i"], a), lambda a, b: min(b, a), -5, [(C["TPLX_ACC_MIN_I64"], (-5) & MASK)]),
        (lambda a, x: max(a, x["i"]), lambda a, b: max(a, b), 2.5, [(C["TPLX_ACC_MAX_F64"], ir.f64_bits(2.5))]),
        (lambda a, x: max(x["f"], a), lambda a, b: max(b, a), -3, [(C["TPLX_ACC_MAX_F64"], ir.f64_bits(-3.0))]),
        (lambda a, x: min(a, x["f"]), lambda a, b: min(a, b), I64_MAX, [(C["TPLX_ACC_MIN_F64"], ir.f64_bits(float(I64_MAX)))]),
        (lambda a, x: x["f"] + a, lambda a, b: b + a, 0, [(C["TPLX_ACC_SUM_F64"], 0)]),
        (lambda a, x: (min(a[0], x["i"]), max(x["f"], a[1]), a[2] + x["i"]),
         lambda a, b: (min(b[0], a[0]), max(a[1], b[1]), b[2] + a[2]), (I64_MAX, -INF, -7),
         [(C["TPLX_ACC_MIN_I64"], I64_MAX), (C["TPLX_ACC_MAX_F64"], ir.f64_bits(-INF)), (C["TPLX_ACC_SUM_I64"], (-7) & MASK)]),
        (AGG6, COMB6, INIT6, [(k, b) for k, b in zip(KINDS6, [1 << 50, (-(1 << 50)) & MASK, 12345, ir.f64_bits(2.0 ** 30),
                                                              ir.f64_bits(-2.0 ** 30), ir.f64_bits(0.25)])]),
    ]
    for agg, comb, init, want in cases[:-1]:
        assert lowered(agg, comb, init, endpoint) == want
    sc = frontend.StageCompiler(TYPES6, NAMES6)
    prog = sc.finish_aggregate(*cases[-1][:3], 100001)
    assert [(a.kind, a.init_bits) for a in prog.accs] == cases[-1][3]
    # a combiner that is not the aggregate's own operation is not lowered
    with pytest.raises(frontend.UnsupportedUDF):
        lowered(lambda a, x: min(a, x["i"]), lambda a, b: max(a, b), 0, endpoint)


EDGE_ROWS = [
    {"a": I64_MAX, "b": I64_MIN, "c": I64_MAX, "d": INF, "e": -INF, "f": 0.5},
    {"a": 3, "b": -3, "c": I64_MAX, "d": SUBNORMAL, "e": -SUBNORMAL, "f": -1 / 64},
    {"a": I64_MIN, "b": I64_MAX, "c": 2, "d": -INF, "e": INF, "f": 2.0 ** 40},
    {"a": -1, "b": 1, "c": I64_MIN, "d": 1.0, "e": -1.0, "f": 3 / 64},
    {"a": I64_MAX, "b": I64_MIN, "c": I64_MIN, "d": -SUBNORMAL, "e": SUBNORMAL, "f": -(2.0 ** 40)},
]


def test_oracle_and_host_fold_match_cpython_reduce_on_value_edges(built):
    from oracle import pyoracle
    prog = k3_program()
    for take in ([0], [1], [0, 1], [1, 3], [0, 2, 4], [0, 1, 2, 3, 4], [4, 3, 2, 1, 0], []):
        rows = [EDGE_ROWS[i] for i in take]
        red = functools.reduce(AGG6, rows, INIT6)
        red = red[:2] + (wrap(red[2]),) + red[3:]
        n = len(rows)
        cols = [ccol([r[k] for r in rows], t) for k, t in zip(NAMES6, TYPES6)] + [ccol([0] * n, T_I64)]
        ora = pyoracle.run_program(prog, cols, n)
        assert ora.acc_seq == bits6(red), take
        assert ora.acc_tree == bits6(red), take
        # the host's partial fold (dataset._acc_combine over device partials) on the same values
        host = list(INIT6)
        for r in rows:
            host = [dataset._acc_combine(k, h, r[name]) for k, h, name in zip(KINDS6, host, NAMES6)]
        assert bits6(host) == bits6(red), take
        assert [dataset._acc_value(k, b) for k, b in zip(KINDS6, bits6(red))] == [float(x) if k in F64_KINDS else x
                                                                                 for k, x in zip(KINDS6, red)]
    assert [dataset._acc_identity_bits(k) for k in KINDS6] == bits6(IDENT6)


def test_oracle_pins_the_device_rule_for_nan_and_signed_zero(built):
    """min(x, a) returns NaN in CPython when the NaN row comes last, and drops it when a value follows; the device (and the
    oracle that restates it) ignores NaN rows in every spelling. Equal zeros keep the one met first (DESIGN §4)."""
    from oracle import pyoracle
    sc = frontend.StageCompiler([T_F64], ["d"])
    prog = sc.finish_aggregate(lambda a, x: (min(x["d"], a[0]), min(a[1], x["d"]), max(a[2], x["d"])),
                               lambda a, b: (min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2])), (INF, INF, -INF), 100001)
    nan = float("nan")
    for vals in ([1.0, nan], [nan, 1.0], [2.0, nan, -1.0]):
        row_first = functools.reduce(lambda a, x: min(x, a), vals, INF)
        acc_first = functools.reduce(lambda a, x: min(a, x), vals, INF)
        assert math.isnan(row_first) == math.isnan(vals[-1]) and not math.isnan(acc_first)
        ora = pyoracle.run_program(prog, [ccol(vals, T_F64)], len(vals))
        lo, hi = float(np.nanmin(vals)), float(np.nanmax(vals))
        assert ora.acc_seq == ora.acc_tree == [ir.f64_bits(lo), ir.f64_bits(lo), ir.f64_bits(hi)]
    ora = pyoracle.run_program(prog, [ccol([0.0, -0.0], T_F64)], 2)
    assert ora.acc_seq == [ir.f64_bits(0.0)] * 2 + [ir.f64_bits(0.0)]
