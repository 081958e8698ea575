"""Option[T] group keys on the device: aggregateByKey and unique() keep None as a group of its own (the reference's null bucket,
PipelineBuilder.cc:1148-1170,1263-1310). None differs from 0, "" and False, a None key's value slot never matters, and the device
result carries the key column with a validity bitmap. Every expectation is a plain Python / numpy group-by written here."""
import struct
import typing
from collections import Counter

import numpy as np
import pytest

import tuplex_b200
import test_gpu_aggregates as agg
import test_gpu_cpp_host as cpp
from tuplex_b200 import backend, dataset, frontend
from tuplex_b200.backend import Block, Column, GpuBackendError
from tuplex_b200.frontend import UnsupportedUDF
from tuplex_b200.ir import C, T_BOOL, T_F64, T_I64, T_STR
from tuplex_b200.pyexec import Op

I64_MIN, I64_MAX = agg.I64_MIN, agg.I64_MAX
NON_UTF8 = b"\xff\xfez"
POOLS = {T_I64: [None, 0, I64_MIN, I64_MAX, -1, 1, 7],
         T_STR: [None, "", "a", "ä", "日本語", NON_UTF8, "None"],
         T_BOOL: [None, False, True]}


def sum_program(in_types, names, key_cols, option_cols=()):
    sc = frontend.StageCompiler(in_types, names, option_cols)
    return sc.finish_hash(key_cols, lambda a, x: a + x["v"], lambda a, b: a + b, 0, 100001)


# =============================================================================================================================
# CPU: front end, descriptor validation, host fold
# =============================================================================================================================
def test_frontend_emits_hidden_companions_for_option_keys(built):
    # keys: k0 Option[i64] (input), s plain str, k1 Option[str] from a UDF that leaves some rows empty
    sc = frontend.StageCompiler([T_I64, T_STR, T_I64], ["k0", "s", "v"], option_cols=[0])
    sc.add_with_column("k1", lambda x: x["s"] if x["v"] > 0 else None, 100001)
    prog = sc.finish_hash(["k0", "s", "k1"], lambda a, x: a + x["v"], lambda a, b: a + b, 0, 100002)
    assert prog.n_keys == 3 and prog.hidden_out_cols == 2
    assert [t for _, t in prog.out_cols] == [T_I64, T_STR, T_STR, T_BOOL, T_BOOL]
    assert prog.out_null_of == [0, 0, 0, 1, 3]
    assert len(prog.accs) == 1
    backend.Stage(prog).close()  # the executor accepts it
    # unique(): every column is a key
    sc = frontend.StageCompiler([T_STR, T_BOOL], ["a", "b"], option_cols=[0, 1])
    prog = sc.finish_hash([0, 1], None, None, None, 100001)
    assert prog.out_null_of == [0, 0, 1, 2] and prog.hidden_out_cols == 2 and not prog.accs
    assert backend.Result(None, backend.Stage(prog), None, hash_result=True).out_types() == [T_STR, T_BOOL]


# sha256 of the descriptors these stages had before Option keys existed: a stage without Option keys keeps its bytes
PLAIN_DESCRIPTORS = ["6221c6ccdb1c513e30176f301954667ac639bdfda4e1d192baaa4855f236448a",
                     "2e079328bcf82f9ccb733e6c0975a39ca9ef0f0fa1248d5cd73cb6a1317adad7",
                     "5cb3f3037ccf0c5082dd667624f2784b07be98a3a71427ae21553cdae2410a18"]


def test_stages_without_option_keys_keep_their_descriptor_bytes(built):
    import hashlib
    types, names = [T_I64, T_STR, T_BOOL, T_F64], ["a", "s", "b", "f"]
    sc = frontend.StageCompiler(types, names)
    p0 = sc.finish_hash(["a"], lambda a, x: (a[0] + x["a"], min(a[1], x["f"])), lambda a, b: (a[0] + b[0], min(a[1], b[1])), (0, 0.0), 100001)
    sc = frontend.StageCompiler(types, names)
    sc.add_with_column("k", lambda x: x["s"][1:] if x["a"] > 0 else "neg", 100001)
    p1 = sc.finish_hash(["k", "b", "a"], lambda a, x: a + x["f"], lambda a, b: a + b, 0.5, 100002)
    sc = frontend.StageCompiler([T_I64, T_STR], ["a", "s"])
    sc.add_map(lambda x: (x["a"] * 2, x["s"].upper()), 100001)
    p2 = sc.finish_hash([0, 1], None, None, None, 100002)
    for p, want in zip((p0, p1, p2), PLAIN_DESCRIPTORS):
        assert p.hidden_out_cols == 0 and not any(p.out_null_of) and len(p.out_cols) == p.n_keys
        assert hashlib.sha256(p.serialize()).hexdigest() == want


def test_none_only_and_f64_keys_are_still_refused(built):
    sc = frontend.StageCompiler([T_I64, T_I64], ["a", "v"])
    sc.add_with_column("k", lambda x: None, 100001)
    with pytest.raises(UnsupportedUDF, match="None for every row"):
        sc.finish_hash(["k"], lambda a, x: a + x["v"], lambda a, b: a + b, 0, 100002)
    with pytest.raises(UnsupportedUDF, match="f64 keys"):
        sum_program([T_F64, T_I64], ["k", "v"], ["k"], option_cols=[0])


def _option_key_program():
    return sum_program([T_I64, T_STR, T_I64], ["k", "s", "v"], ["k", "s"], option_cols=[0])


def test_descriptor_validation_of_key_companions(built):
    prog = _option_key_program()
    assert prog.out_null_of == [0, 0, 1]
    backend.Stage(prog).close()

    def rejected(mutate):
        p = _option_key_program()
        mutate(p)
        with pytest.raises(GpuBackendError, match="companion"):
            backend.Stage(p)

    rejected(lambda p: setattr(p, "hidden_out_cols", 0))                                    # visible
    rejected(lambda p: p.out_cols.__setitem__(2, (p.out_cols[2][0], T_I64)))                # not bool
    rejected(lambda p: p.out_null_of.__setitem__(2, 3))                                     # points past n_keys (at itself)
    rejected(lambda p: p.out_null_of.__setitem__(2, 4))                                     # past every column (an accumulator)
    rejected(lambda p: p.out_null_of.__setitem__(0, 1))                                     # on a key column

    def twice(p):  # two companions of one key
        p.out_cols.append(p.out_cols[2])
        p.out_null_of.append(1)
        p.hidden_out_cols = 2
    rejected(twice)

    def on_aggregate(p):  # the AGGREGATE endpoint has no key columns to point at
        p.endpoint = C["TPLX_EP_AGGREGATE"]
        p.n_keys = 0
    rejected(on_aggregate)


class _FakeResult:
    def __init__(self, cols):
        self._cols = cols

    def columns(self):
        return self._cols

    def free(self):
        pass


class _FakeStage:
    def __init__(self, cols):
        self._cols = cols

    def hash_finish(self, dev):
        return _FakeResult(self._cols)


def test_host_fold_puts_interpreter_rows_with_none_keys_into_the_device_none_group(built):
    """A device result with a None key plus fallback rows whose key is None: one None group, aggregated over both."""
    prog = sum_program([T_I64, T_I64], ["k", "v"], ["k"], option_cols=[0])
    end = Op("aggregateByKey", udf=lambda a, x: a + x["v"], columns=["k"], extra=(lambda a, b: a + b, 0))
    plan = dataset._StagePlan(prog, [], end, ["k", "v"], False, None)
    keys = Column.from_values([None, 0, 5], T_I64)
    assert keys.valid is not None
    dev_cols = [keys, Column(T_I64, np.array([10, 20, 30], np.int64))]
    st = dataset._Shard(None)
    st.fallback = [(100, (None, 1)), (101, (None, 2)), (102, (0, 4)), (103, ("x", 8))]
    rows, names = dataset._hash_endpoint(plan, _FakeStage(dev_cols), st, [0], ["k", "v"], Counter())
    assert rows == [(None, 13), (0, 24), (5, 30), ("x", 8)]
    assert names == ["k", None]


# =============================================================================================================================
# GPU through the C ABI
# =============================================================================================================================
def opt_col(vals, t, rng, bitmap=True) -> Column:
    """Column of `vals` (None = missing). The value slot under None holds different nonzero junk on every row: the device must never
    look at it. bitmap=False: no validity bitmap at all (only for columns without None)."""
    present = np.array([v is not None for v in vals], bool)
    if t == T_STR:
        enc = [(v if isinstance(v, bytes) else v.encode()) if v is not None else b"junk%d" % int(rng.integers(1, 1 << 40)) for v in vals]
        offsets = np.zeros(len(enc) + 1, np.uint32)
        np.cumsum([len(b) for b in enc], out=offsets[1:])
        c = Column(T_STR, np.frombuffer(b"".join(enc), np.uint8).copy(), offsets)
    else:
        junk = rng.integers(1, 1 << 62, len(vals))
        c = Column(t, np.array([int(v) if v is not None else int(j) for v, j in zip(vals, junk.tolist())], np.int64))
    if bitmap:
        c.valid = backend.pack_valid(present)
    else:
        assert present.all()
    return c


def ref_key(v):
    """A key as the device result gives it back (strings are decoded with errors='replace')."""
    return v.decode("utf-8", "replace") if isinstance(v, bytes) else v


def run6(st, v, key_cols, n):
    return st.run_host(0, [agg.ccol(v[k], t) for k, t in zip(agg.NAMES6, agg.TYPES6)] + key_cols, n)


def prog6(key_names, key_types, option=True):
    n6 = len(agg.NAMES6)
    sc = frontend.StageCompiler(agg.TYPES6 + list(key_types), agg.NAMES6 + list(key_names),
                                option_cols=list(range(n6, n6 + len(key_names))) if option else ())
    return sc.finish_hash(list(key_names), agg.AGG6, agg.COMB6, agg.INIT6, 100001)


def check_groups(res, keys, rows, nk):
    got = agg.fetch_groups(res, nk)
    want = {k: agg.bits6(agg.finish6(b)) for k, b in agg.group_reference(keys, rows).items()}
    assert got.keys() == want.keys()
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, f"{len(bad)} of {len(want)} groups differ, e.g. {bad[0]}: {got[bad[0]]} != {want[bad[0]]}"
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("kt", [T_I64, T_STR, T_BOOL], ids=["i64", "str", "bool"])
def test_single_option_key_value_edges_two_blocks(gpu, kt):
    """None next to 0 / "" / False / INT64_MIN / INT64_MAX / non-UTF-8 bytes, every accumulator kind on every group, over four
    blocks into one table: keys with None, every key None, a bitmap without None, no bitmap."""
    st = backend.Stage(prog6(["k"], [kt]))
    rng = np.random.default_rng(40 + kt)
    pool = POOLS[kt]
    keys, rows = [], []
    for mode in ("mixed", "all_none", "bitmap_no_none", "no_bitmap"):
        n = 50_000 + 311 * len(keys) % 1000
        if mode == "mixed":
            kv = [pool[i] for i in rng.integers(0, len(pool), n)]
        elif mode == "all_none":
            kv = [None] * n
        else:
            kv = [pool[i] for i in rng.integers(1, len(pool), n)]
        v = agg.with_edges(rng, agg.values6(rng, n), n)
        run6(st, v, [opt_col(kv, kt, rng, bitmap=mode != "no_bitmap")], n).info
        keys += [(ref_key(k),) for k in kv]
        rows += agg.rows_of(v, range(n))
    res = st.hash_finish(0)
    got = check_groups(res, keys, rows, 1)
    assert (None,) in got and len(got) == len(pool)
    kc = res.columns()[0]
    present = kc.present()
    assert present is not None and int((~present).sum()) == 1
    # the placeholder under None: 0 / empty string (DESIGN §2)
    i = int(np.flatnonzero(~present)[0])
    if kt == T_STR:
        assert kc.offsets[i] == kc.offsets[i + 1]
    else:
        assert kc.data[i] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["first", "middle", "last", "max_keys"])
def test_multi_column_option_keys(gpu, where):
    """(None, 1) != (0, 1) != (None, 2): the Option key first, in the middle, last, and TPLX_MAX_KEYS keys that are all Option."""
    rng = np.random.default_rng(50)
    if where == "max_keys":
        types = [[T_I64, T_STR, T_BOOL][i % 3] for i in range(C["TPLX_MAX_KEYS"])]
        opt = list(range(len(types)))
    else:
        types = [T_I64, T_STR, T_BOOL]
        opt = [{"first": 0, "middle": 1, "last": 2}[where]]
    names = ["k%d" % i for i in range(len(types))]
    n6 = len(agg.NAMES6)
    sc = frontend.StageCompiler(agg.TYPES6 + types, agg.NAMES6 + names, option_cols=[n6 + i for i in opt])
    st = backend.Stage(sc.finish_hash(names, agg.AGG6, agg.COMB6, agg.INIT6, 100001))
    n = 120_000
    small = {T_I64: [None, 0, 1, 2], T_STR: [None, "", "a"], T_BOOL: [None, False, True]}
    kv = []
    for i, t in enumerate(types):
        pool = small[t] if i in opt else small[t][1:]
        kv.append([pool[j] for j in rng.integers(0, len(pool), n)])
    v = agg.values6(rng, n)
    run6(st, v, [opt_col(kv[i], t, rng, bitmap=i in opt) for i, t in enumerate(types)], n).info
    keys = list(zip(*kv))
    check_groups(st.hash_finish(0), keys, agg.rows_of(v, range(n)), len(types))


def _numpy_check(res, keys, none, v):
    """Device result vs numpy: the None group is keyed -1 on both sides (data keys are >= 0)."""
    ref = np.where(none, -1, keys)
    uk, out = agg.numpy_groups(ref, v)
    cols = res.columns()
    present = cols[0].present()
    assert present is not None
    dk = np.where(present, cols[0].data, -1)
    order = np.argsort(dk, kind="stable")
    assert np.array_equal(dk[order], uk), f"{len(dk)} keys emitted, {len(uk)} expected"
    want = agg.numpy_finish_bits(out)
    for i in range(6):
        got = cols[1 + i].data[order].view(np.uint64)
        assert np.array_equal(got, want[i]), f"accumulator {i}: {int((got != want[i]).sum())} of {len(uk)} groups differ"


@pytest.mark.gpu
def test_growth_mid_block_with_none_key_rows_in_the_overflow_list(gpu):
    n = 400_000
    rng = np.random.default_rng(51)
    keys = np.arange(n, dtype=np.int64) * 7919
    none = rng.random(n) < 0.1
    st = backend.Stage(prog6(["k"], [T_I64]))
    st.hash_reserve(0, 1000)
    v = agg.values6(rng, n)
    run6(st, v, [opt_col([None if z else int(k) for k, z in zip(keys.tolist(), none.tolist())], T_I64, rng)], n).info
    _numpy_check(st.hash_finish(0), keys, none, v)


@pytest.mark.gpu
def test_high_cardinality_with_none_rows_switches_off_the_buckets(gpu):
    n = 3_000_000
    rng = np.random.default_rng(52)
    keys = np.arange(n, dtype=np.int64) + 1000
    none = rng.random(n) < 0.1
    col = Column(T_I64, np.where(none, rng.integers(1, 1 << 62, n), keys), None, backend.pack_valid(~none))
    st = backend.Stage(prog6(["k"], [T_I64]))
    v = agg.values6(rng, n)
    run6(st, v, [col], n).info
    _numpy_check(st.hash_finish(0), keys, none, v)


@pytest.mark.gpu
def test_exception_rows_past_the_buffer_with_none_keys(gpu):
    n = 300_000
    rng = np.random.default_rng(53)
    num, bad, s = agg.dirty_ints(rng, n)
    kv = [None if r < 0.2 else int(k) for r, k in zip(rng.random(n).tolist(), rng.integers(0, 97, n).tolist())]
    sc = frontend.StageCompiler([T_STR, T_I64], ["s", "k"], option_cols=[1])
    sc.add_with_column("v", lambda x: int(x["s"]), 100001)
    st = backend.Stage(sc.finish_hash(["k"], lambda a, x: a + x["v"], lambda a, b: a + b, 0, 100002))
    res = st.run_host(0, [agg.ccol(s, T_STR), opt_col(kv, T_I64, rng)], n)
    exc = res.exceptions()
    assert len(exc) == int(bad.sum()) > max(4096, n // 32)
    assert sorted(exc["row"].tolist()) == np.flatnonzero(bad).tolist()
    want = {}
    for k, q, b in zip(kv, num.tolist(), bad.tolist()):
        if not b:
            want[k] = want.get(k, 0) + q
    cols = st.hash_finish(0).columns()
    got = dict(zip(cols[0].to_values(), cols[1].data.tolist()))
    assert len(got) == len(cols[0]) and got == want and None in got


@pytest.mark.gpu
def test_raw_export_packed_bitmaps_and_merge(gpu):
    """The single-device half of the exchange: stage A exports raw partials whose key columns carry bitmaps, stage B merges that
    packed block into its own table and finishes; also a merge into an empty stage and a packed key column without a bitmap."""
    n = 120_000
    rng = np.random.default_rng(54)
    v = agg.with_edges(rng, agg.values6(rng, n), n)
    ks = [POOLS[T_STR][i] for i in rng.integers(0, len(POOLS[T_STR]), n)]
    kk = [[None, 0, 1, -5][i] for i in rng.integers(0, 4, n)]
    prog = prog6(["s", "k"], [T_STR, T_I64])
    h = n // 2 + 77

    def cols(lo, hi):
        return [opt_col(ks[lo:hi], T_STR, rng), opt_col(kk[lo:hi], T_I64, rng)]

    keys = [(ref_key(a), b) for a, b in zip(ks, kk)]
    a = backend.Stage(prog)
    run6(a, {k: x[:h] for k, x in v.items()}, cols(0, h), h).info
    raw = a.hash_finish(0, raw=True)
    first = agg.group_reference(keys[:h], agg.rows_of(v, range(h)))
    assert agg.fetch_groups(raw, 2) == {k: agg.bits6(b) for k, b in first.items()}
    rcols = raw.columns()
    assert rcols[0].valid is not None and rcols[1].valid is not None
    block = Block.upload(0, rcols, int(raw.info.n_out_rows))
    b = backend.Stage(prog)
    run6(b, {k: x[h:] for k, x in v.items()}, cols(h, n), n - h).info
    b.hash_merge(block)
    want = {k: agg.bits6(agg.finish6(x)) for k, x in agg.group_reference(keys, agg.rows_of(v, range(n))).items()}
    assert agg.fetch_groups(b.hash_finish(0), 2) == want
    c = backend.Stage(prog)
    c.hash_merge(block)
    assert agg.fetch_groups(c.hash_finish(0), 2) == {k: agg.bits6(agg.finish6(x)) for k, x in first.items()}
    # a packed block whose Option key columns carry no bitmap holds no None
    sel = [i for i, (x, y) in enumerate(zip(rcols[0].to_values(), rcols[1].to_values())) if x is not None and y is not None]
    idx = np.array(sel)
    plain = [Column.from_values([rcols[0].to_values()[i] for i in sel], T_STR), Column(T_I64, rcols[1].data[idx])] + \
            [Column(col.type, col.data[idx]) for col in rcols[2:]]
    d = backend.Stage(prog)
    d.hash_merge(Block.upload(0, plain, len(sel)))
    got = agg.fetch_groups(d.hash_finish(0), 2)
    assert got == {k: agg.bits6(agg.finish6(x)) for k, x in first.items() if None not in k}
    # a bitmap on a column the stage cannot see as None is refused
    with pytest.raises(GpuBackendError, match="validity bitmap"):
        backend.Stage(prog6(["s", "k"], [T_STR, T_I64], option=False)).hash_merge(block)


@pytest.mark.gpu
def test_cpp_host_hash_stage_with_none_keys(gpu, tmp_path):
    """GpuBackend's hash endpoint: the partitions K5 writes carry the None keys in the row bitmap (Serializer.cc:1041-1059)."""
    n = 30_000
    rng = np.random.default_rng(55)
    a = rng.integers(-40, 40, n)
    vv = rng.integers(-3, 10, n)
    sc = frontend.StageCompiler([T_I64, T_I64], ["a", "v"])
    sc.add_with_column("k", lambda x: x["a"] if x["v"] > 0 else None, 100001)
    prog = sc.finish_hash(["k"], lambda acc, x: acc + (x["a"] * 3 + x["v"]), lambda p, q: p + q, 0, 100002)
    assert prog.hidden_out_cols == 1
    info, prefix, _ = cpp._run_host(tmp_path, prog, [Column(T_I64, a.astype(np.int64)), Column(T_I64, vv.astype(np.int64))], n,
                                    [T_I64, T_I64], 16 << 10, "0,0")
    got = []
    for i in range(info["hash_partitions"]):
        part = open(f"{prefix}.hash{i}", "rb").read()
        rows = struct.unpack_from("<q", part, 0)[0]
        p = 8
        for _ in range(rows):  # row: 8-byte bitmap (bit 0: the key is None), key slot, sum slot
            bits, key, s = struct.unpack_from("<Qqq", part, p)
            got.append((None if bits & 1 else key, s))
            p += 24
    want = {}
    for x, y in zip(a.tolist(), vv.tolist()):
        k = x if y > 0 else None
        want[k] = want.get(k, 0) + x * 3 + y
    assert len(got) == len(want) == info["out_rows"]
    assert dict(got) == want and None in want


# =============================================================================================================================
# GPU through Context: each source of an Option key, unique(), the interpreter path joining the None group
# =============================================================================================================================
@pytest.fixture
def ctx(gpu):
    return tuplex_b200.Context({"tuplex.gpu.blockRows": 20_000})


def groups_of(rows):
    d = dict(rows)
    assert len(d) == len(rows), "a group was emitted twice"
    return d


@pytest.mark.gpu
def test_context_parallelize_with_none_keys(ctx):
    rng = np.random.default_rng(60)
    n = 70_000
    kv = [[None, 0, 3, -3][i] for i in rng.integers(0, 4, n)]
    sv = [["", "x", None, "None"][i] for i in rng.integers(0, 4, n)]
    vv = rng.integers(-100, 100, n).tolist()
    rows = list(zip(kv, sv, vv))
    got = ctx.parallelize(rows, columns=["k", "s", "v"]).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["k"]).collect()
    assert ctx.metrics.rows_in > 0
    want = {}
    for k, _, v in rows:
        want[k] = want.get(k, 0) + v
    assert groups_of(got) == want and got[0][0] is None  # None sorts first
    got2 = ctx.parallelize(rows, columns=["k", "s", "v"]).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["s", "k"]).collect()
    want2 = {}
    for k, s, v in rows:
        want2[(s, k)] = want2.get((s, k), 0) + v
    assert {(s, k): v for s, k, v in got2} == want2 and len(got2) == len(want2) == 16
    ds = ctx.parallelize(rows, columns=["k", "s", "v"]).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["k"])
    assert ds.types[0] == typing.Optional[int]


@pytest.mark.gpu
def test_context_udf_that_leaves_the_key_empty(ctx):
    """map that returns x['a'] if x['b'] > 0 else None: the value slot holds x['a'] under None, and must not split the None group."""
    rng = np.random.default_rng(61)
    n = 60_000
    rows = list(zip(rng.integers(0, 50, n).tolist(), rng.integers(-5, 5, n).tolist(), rng.integers(0, 1000, n).tolist()))
    ds = ctx.parallelize(rows, columns=["a", "b", "v"]).withColumn("k", lambda x: x["a"] if x["b"] > 0 else None)
    got = ds.aggregateByKey(lambda p, q: p + q, lambda acc, x: acc + x["v"], 0, ["k"]).collect()
    assert ctx.metrics.rows_in > 0
    want = {}
    for a, b, v in rows:
        k = a if b > 0 else None
        want[k] = want.get(k, 0) + v
    assert groups_of(got) == want


@pytest.mark.gpu
def test_context_left_join_then_group_by_a_right_column(ctx):
    rng = np.random.default_rng(62)
    L = [(int(k), int(v)) for k, v in zip(rng.integers(0, 400, 30_000), rng.integers(0, 100, 30_000))]
    R = [(int(k), "c%d" % (k % 7)) for k in range(0, 300, 2)]
    ds = ctx.parallelize(L, columns=["k", "v"]).leftJoin(ctx.parallelize(R, columns=["k", "city"]), "k", "k")
    got = ds.aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["city"]).collect()
    assert ctx.metrics.rows_in > 0
    city = dict(R)
    want = {}
    for k, v in L:
        c = city.get(k)
        want[c] = want.get(c, 0) + v
    assert groups_of(got) == want and None in want


@pytest.mark.gpu
def test_context_unique_with_none_in_each_column(ctx):
    rng = np.random.default_rng(63)
    n = 50_000
    rows = [([None, 1, 0][i], [None, "", "a"][j], [None, False, True][m])
            for i, j, m in zip(rng.integers(0, 3, n), rng.integers(0, 3, n), rng.integers(0, 3, n))]
    got = ctx.parallelize(rows).unique().collect()
    assert ctx.metrics.rows_in > 0
    assert len(got) == len(set(got)) == len(set(rows)) == 27 and set(got) == set(rows)
    assert got[0] == (None, None, None)


@pytest.mark.gpu
def test_context_resolved_and_fallback_rows_join_the_none_group(ctx):
    """Rows whose UDF raises on the device and is resolved, and fallback rows of another type, all with None keys."""
    rows = [(None, 5), (1, 2), (None, 0), (1, 0), (None, 4), (2, 1)] * 3000 + [(None, "x"), (3, "y"), ("s", 1), (None, 4.0)]

    def fold(row):
        k, v = row
        try:
            q = 100 // v
        except ZeroDivisionError:
            q = -7
        except TypeError:
            return None
        return k, q

    ds = ctx.parallelize(rows, columns=["k", "v"]).map(lambda x: (x["k"], 100 // x["v"])).resolve(ZeroDivisionError, lambda x: (x["k"], -7))
    got = ds.aggregateByKey(lambda a, b: a + b, lambda a, x: a + x[1], 0, [0]).collect()
    assert ctx.metrics.rows_in > 0 and ctx.metrics.exceptions > 0
    want = {}
    for r in rows:
        t = fold(r)
        if t is not None:
            want[t[0]] = want.get(t[0], 0) + t[1]
    assert groups_of(got) == want


@pytest.mark.gpu
def test_context_two_devices_exchange_option_keys(gpu):
    """tuplex.gpu.devices=0,1: the hash exchange sends each Option key column's bitmap next to its data."""
    if backend.device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(64)
    n = 100_000
    rows = list(zip([[None, "", "a", "b"][i] for i in rng.integers(0, 4, n)], rng.integers(-9, 9, n).tolist(),
                    rng.integers(0, 100, n).tolist()))
    two = tuplex_b200.Context({"tuplex.gpu.blockRows": 7000, "tuplex.gpu.devices": "0,1"})
    got = two.parallelize(rows, columns=["s", "k", "v"]).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["s", "k"]).collect()
    want = {}
    for s, k, v in rows:
        want[(s, k)] = want.get((s, k), 0) + v
    assert {(s, k): v for s, k, v in got} == want and len(got) == len(want)


@pytest.mark.gpu
@pytest.mark.parametrize("none_first", [True, False], ids=["none_on_device0", "none_on_device1"])
def test_context_two_devices_rank_without_keys_of_its_own(gpu, none_first):
    """Input sorted by key: each device's blocks hold a single key, None on one device and a string on the other. Over the four
    strings, some is owned by the device that holds None, so the other device owns none of its own keys and receives only the None
    group (with its bitmap) from its peer."""
    if backend.device_count() < 2:
        pytest.skip("needs two GPUs")
    half = 14_000
    two = tuplex_b200.Context({"tuplex.gpu.blockRows": 7000, "tuplex.gpu.devices": "0,1"})
    for other in ("a", "b", "c", "d"):
        keys = [None] * half + [other] * half if none_first else [other] * half + [None] * half
        rows = [(k, i % 10) for i, k in enumerate(keys)]
        got = two.parallelize(rows, columns=["s", "v"]).aggregateByKey(lambda a, b: a + b, lambda a, x: a + x["v"], 0, ["s"]).collect()
        want = {None: sum(v for k, v in rows if k is None), other: sum(v for k, v in rows if k == other)}
        assert groups_of(got) == want, other
