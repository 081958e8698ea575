"""Parity proper: the CUDA path through the C ABI vs the CPU oracle on the same seeded inputs, bit-exact
(integer / string / per-row f64; f64 aggregates vs the oracle's same reduction tree and within a bound of
the sequential reference order)."""
import hashlib

import numpy as np
import pytest

from tuplex_b200 import backend, frontend, ir, workloads
from tuplex_b200.backend import Column
from tuplex_b200.ir import T_F64, T_I64, T_STR
from oracle import pyoracle
from helpers import assert_result_equals_oracle, run_both

pytestmark = pytest.mark.gpu


def test_c1_map_filter(gpu):
    x = np.arange(1, 1_000_001, dtype=np.int64)
    prog = workloads.c1_program()
    st, res, ora = run_both(prog, [Column(T_I64, x)], len(x))
    assert_result_equals_oracle(res, ora, "C1")
    assert int(res.info.n_out_rows) == 500_000
    assert np.array_equal(res.column(0).data, pyoracle.c1(x))


@pytest.mark.parametrize("n", [0, 1, 31, 255, 256, 257, 4095, 4096, 4097, 100_003])
def test_ragged_sizes(gpu, n):
    rng = np.random.default_rng(n)
    x = rng.integers(-10**6, 10**6, n, dtype=np.int64)
    prog = workloads.c1_program()
    st, res, ora = run_both(prog, [Column(T_I64, x)], n)
    assert_result_equals_oracle(res, ora, f"n={n}")


def test_int_arith_and_exceptions(gpu):
    rng = np.random.default_rng(7)
    n = 50_000
    a = rng.integers(-1000, 1000, n, dtype=np.int64)
    b = rng.integers(-5, 6, n, dtype=np.int64)  # ~9% zeros -> ZeroDivisionError rows
    sc = frontend.StageCompiler([T_I64, T_I64], ["a", "b"])
    sc.add_map(lambda x: (x['a'] // x['b'], x['a'] % x['b'], x['a'] * x['b'] - 3, x['a'] / x['b']), 100001)
    sc.add_filter(lambda x: x[1] != 2, 100002)
    prog = sc.finish_memory()
    st, res, ora = run_both(prog, [Column(T_I64, a), Column(T_I64, b)], n, first_row_no=17)
    assert len(ora.exceptions) > 1000
    assert set(ora.exceptions["code"].tolist()) == {136}
    assert_result_equals_oracle(res, ora, "int arith")


def test_float_ops_bit_exact(gpu):
    rng = np.random.default_rng(11)
    n = 40_000
    a = rng.normal(0, 1e3, n)
    b = rng.normal(0, 10, n)
    b[::97] = 0.0
    sc = frontend.StageCompiler([T_F64, T_F64], ["a", "b"])
    sc.add_map(lambda x: (x['a'] * x['b'] + 0.1, x['a'] / x['b'], x['a'] % x['b'], x['a'] - x['b'] * 3, int(x['a'])), 100001)
    sc.add_filter(lambda x: x[0] < 1e4 and x[1] != 7.0, 100002)
    prog = sc.finish_memory()
    st, res, ora = run_both(prog, [Column(T_F64, a), Column(T_F64, b)], n)
    assert_result_equals_oracle(res, ora, "float ops")


def test_q6_golden_and_tree(gpu):
    cols = workloads.load_lineitem_fixture()
    n = len(cols[0].data)
    prog = workloads.q6_program()
    st, res, ora = run_both(prog, cols, n)
    bits = res.aggregate_bits()
    assert bits == ora.acc_tree, "aggregate differs from the oracle's same reduction tree"
    got = ir.bits_f64(bits[0])
    seq = ir.bits_f64(ora.acc_seq[0])
    assert repr(seq) == "1193053.2252999984"  # gtest golden (TPCH.cc:85-97), sequential order
    assert abs(got - 1193053.2252999984) <= 1e-4  # the reference test's own tolerance
    assert seq == pyoracle.q6(cols[0].data, cols[1].data, cols[2].data, cols[3].data)


def test_q6_synthetic_large(gpu):
    n = 5_000_000
    cols = workloads.gen_lineitem(n, seed=42)
    prog = workloads.q6_program()
    st, res, ora = run_both(prog, cols, n)
    assert res.aggregate_bits() == ora.acc_tree
    got, seq = ir.bits_f64(res.aggregate_bits()[0]), ir.bits_f64(ora.acc_seq[0])
    # |tree - sequential| <= n_qualifying * eps * sum|x|
    assert abs(got - seq) <= 1e-9 * abs(seq)


def test_zillow_fixture_md5(gpu):
    cols, n = workloads.load_zillow_fixture()
    prog = workloads.zillow_program()
    st, res, ora = run_both(prog, cols, n)
    assert_result_equals_oracle(res, ora, "zillow")
    vals = [c.to_values() for c in res.columns()]
    txt = workloads.rows_to_csv(vals, workloads.ZILLOW_OUT)
    assert hashlib.md5(txt).hexdigest() == "4d5ca0263b1a5058341a369116dee83a"
    assert txt == workloads.zillow_golden_csv()


def test_zillow_replicated_cycles(gpu):
    cols, n0 = workloads.load_zillow_fixture()
    n = 10 * n0 + 1234
    big = workloads.replicate(cols, n0, n)
    prog = workloads.zillow_program()
    st = backend.Stage(prog)
    res = st.run_host(0, big, n)
    vals = [c.to_values() for c in res.columns()]
    golden = workloads.zillow_golden_csv().decode().split("\n")[1:-1]
    per = 577
    assert int(res.info.n_out_rows) >= 10 * per
    one = workloads.rows_to_csv([v[:per] for v in vals], None).decode().split("\n")[:-1]
    assert one == golden
    # every full cycle reproduces the golden rows (idempotence across tile boundaries)
    for k in (1, 5, 9):
        cyc = workloads.rows_to_csv([v[k * per:(k + 1) * per] for v in vals], None).decode().split("\n")[:-1]
        assert cyc == golden


def test_string_ops_and_exceptions(gpu):
    rng = np.random.default_rng(5)
    words = ["12", " 7 ", "-3", "x9", "", "  ", "-", "0042", "1e3", "9 9", "77\t", "+5", "123456789012"]
    n = 20_000
    s = [words[i] for i in rng.integers(0, len(words), n)]
    t = ["Ab,c" * int(k) for k in rng.integers(0, 4, n)]
    sc = frontend.StageCompiler([T_STR, T_STR], ["s", "t"])
    sc.add_with_column("v", lambda x: int(x['s']), 100001)
    sc.add_with_column("u", lambda x: x['t'].replace(',', '').upper() + '_' + x['s'].strip(), 100002)
    sc.add_with_column("w", lambda x: x['t'][0] + x['t'][-1:], 100003)
    sc.add_filter(lambda x: x['v'] != 12 and 'B' in x['u'], 100004)
    sc.add_with_column("z", lambda x: '%05d' % x['v'] + ('%d' % len(x['u'])), 100005)
    prog = sc.finish_memory()
    cols = [Column.from_values(s, T_STR), Column.from_values(t, T_STR)]
    st, res, ora = run_both(prog, cols, n, first_row_no=3)
    codes = set(ora.exceptions["code"].tolist())
    assert 135 in codes and 111 in codes  # ValueError from int(), IndexError from t[0] on ''
    assert_result_equals_oracle(res, ora, "string ops")


def test_exception_partition_and_row_format(gpu):
    rng = np.random.default_rng(3)
    n = 30_000
    a = rng.integers(-50, 50, n, dtype=np.int64)
    s = ["v%d" % v for v in a]
    sc = frontend.StageCompiler([T_I64, T_STR], ["a", "s"])
    sc.add_with_column("q", lambda x: 100 // x['a'], 100001)
    sc.add_filter(lambda x: x['q'] != 5, 100002)
    prog = sc.finish_memory()
    cols = [Column(T_I64, a), Column.from_values(s, T_STR)]
    st, res, ora = run_both(prog, cols, n)
    assert_result_equals_oracle(res, ora, "exc")
    # K2: exception partition bytes == oracle restatement of IExceptionableTask.h:22-36
    assert res.exception_partition() == pyoracle.exception_partition(cols, ora.exceptions)
    # K5 (columns -> Partition bytes), small partitions force many splits
    class OC:  # oracle-side view of the oracle's output columns
        def __init__(self, t, d, o): self.type, self.data, self.offsets = t, d, o
    ocols = [OC(t, d, o) for t, d, o in ora.columns]
    for psize in (4096, 1 << 20):
        assert res.partitions(psize) == pyoracle.to_partitions(ocols, ora.n_out, psize)


def test_partitions_roundtrip_input(gpu):
    """K5 the other way: reference-format partitions -> column block -> same stage result."""
    cols, n0 = workloads.load_zillow_fixture()
    n = 5000
    small = [c.slice(0, n) for c in cols]
    parts = pyoracle.to_partitions(small, n, 64 << 10)
    assert len(parts) > 5
    blk = backend.Block.from_partitions(0, parts, workloads.ZILLOW_TYPES)
    assert blk.n_rows == n
    prog = workloads.zillow_program()
    st = backend.Stage(prog)
    res = st.run(blk)
    ora = pyoracle.run_program(prog, small, n)
    assert_result_equals_oracle(res, ora, "from partitions")


def test_hash_aggregate_i64_and_str(gpu):
    n = 300_000
    cols = workloads.gen_keyed(n, 5000, seed=9)
    prog = workloads.keyed_program()
    st = backend.Stage(prog)
    res = st.run_host(0, cols, n)
    res.info
    fin = st.hash_finish(0)
    ora = pyoracle.run_program(prog, cols, n)
    got = dict(zip(fin.column(0).to_values(), fin.column(1).to_values()))
    want = dict(zip(ora.values(0), ora.values(1)))
    assert got == want
    # golden of AggregateTest.cc:249-261 (values scaled x2500 :307-324)
    rows = [(1, "abc", 0), (2, "xyz", 1), (4, "xyz", 2), (3, "abc", -1)] * 2500
    c = [Column.from_values([r[0] for r in rows], T_I64), Column.from_values([r[1] for r in rows], T_STR),
         Column.from_values([r[2] for r in rows], T_I64)]
    sc = frontend.StageCompiler([T_I64, T_STR, T_I64], ["col0", "col1", "col2"])
    p2 = sc.finish_hash(["col1"], lambda a, x: a + x[0] * x[2], lambda a, b: a + b, 0, 100001)
    st2 = backend.Stage(p2)
    st2.run_host(0, c, len(rows)).info
    f2 = st2.hash_finish(0)
    assert sorted(zip(f2.column(0).to_values(), f2.column(1).to_values())) == [("abc", -7500), ("xyz", 25000)]


def test_hash_table_growth(gpu):
    n = 400_000
    keys = np.arange(n, dtype=np.int64) * 7919
    vals = np.ones(n, dtype=np.int64)
    sc = frontend.StageCompiler([T_I64, T_I64], ["k", "v"])
    prog = sc.finish_hash(["k"], lambda a, x: a + x[1], lambda a, b: a + b, 0, 100001)
    st = backend.Stage(prog)
    st.hash_reserve(0, 1000)  # far too small: forces overflow-row retry + rehash
    st.run_host(0, [Column(T_I64, keys), Column(T_I64, vals)], n).info
    st.run_host(0, [Column(T_I64, keys), Column(T_I64, vals)], n).info
    fin = st.hash_finish(0)
    k, v = fin.column(0).data, fin.column(1).data
    assert len(k) == n and set(v.tolist()) == {2}
    assert np.array_equal(np.sort(k), keys)


def test_prefilter_exception_numbering(gpu):
    """Selective pipeline -> prefilter launch + dense launch; exceptions raised in either launch must be
    numbered exactly like one TransformTask numbers them (rows written + exceptions so far)."""
    rng = np.random.default_rng(21)
    words = ["7", "12", "x", "30", "", "9", "21", "70", "7 ", "5"]
    n = 60_000
    s = [words[i] for i in rng.integers(0, len(words), n)]
    sc = frontend.StageCompiler([T_STR], ["s"])
    sc.add_with_column("v", lambda x: int(x['s']), 100001)                    # ValueError rows (prefilter launch)
    sc.add_filter(lambda x: x['v'] % 3 != 0, 100002)
    sc.add_with_column("w", lambda x: ('%03d' % (100 // (x['v'] - 7))) + x['s'].replace('7', 'seven'), 100003)  # ZeroDivisionError
    sc.add_with_column("u", lambda x: x['w'].upper() + '!' + x['s'], 100004)
    prog = sc.finish_memory()
    assert prog.prefilter is not None and prog.hidden_out_cols == 1
    cols = [Column.from_values(s, T_STR)]
    st, res, ora = run_both(prog, cols, n, first_row_no=5)
    codes = set(ora.exceptions["code"].tolist())
    assert codes == {135, 136}
    assert_result_equals_oracle(res, ora, "prefilter exceptions")
    assert res.exception_partition() == pyoracle.exception_partition(cols, ora.exceptions)
    # same stage without the prefilter hint gives the same answer
    sc2 = frontend.StageCompiler([T_STR], ["s"])
    for name, a in sc.oplog:
        getattr(sc2, name)(*a)
    p2 = sc2.finish_memory(prefilter=False)
    assert p2.prefilter is None
    st2, res2, ora2 = run_both(p2, cols, n, first_row_no=5)
    assert_result_equals_oracle(res2, ora, "no prefilter")


def test_fused_scan_aggregate_matches_vm_and_oracle(gpu):
    """K3f (closed-form streaming kernel) vs the VM path (TPLX_NO_FUSED=1) vs the oracle: identical bits."""
    import os
    n = 1_000_003
    cols = workloads.gen_lineitem(n, seed=7)
    progs = []
    progs.append(workloads.q6_program())
    sc = frontend.StageCompiler(workloads.Q6_TYPES, workloads.Q6_COLS)
    sc.add_filter(lambda x: 0.06 - 0.01 <= x['l_discount'] <= 0.06 + 0.01 and x['l_quantity'] < 24, 100001)
    sc.add_filter(lambda x: x['l_shipdate'] >= 19940101, 100002)
    progs.append(sc.finish_aggregate(lambda a, x: (a[0] + 1, a[1] + x[0], a[2] + x[1]), lambda a, b: (a[0] + b[0], a[1] + b[1], a[2] + b[2]),
                                     (0, 0, 0.0), 100003))
    sc = frontend.StageCompiler(workloads.Q6_TYPES, workloads.Q6_COLS)
    sc.add_filter(lambda x: x['l_quantity'] == 7, 100001)
    sc.add_filter(lambda x: x['l_quantity'] < 20.5, 100002)   # i64 column against a float constant -> f64 compare
    progs.append(sc.finish_aggregate(lambda a, x: a + x[0] * x[3], lambda a, b: a + b, 0, 100003))
    sc = frontend.StageCompiler(workloads.Q6_TYPES, workloads.Q6_COLS)
    progs.append(sc.finish_aggregate(lambda a, x: a + x[0] * x[2], lambda a, b: a + b, 0.0, 100001))  # no filter, i64 * f64
    for i, prog in enumerate(progs):
        assert prog.fused is not None, f"program {i} should match the closed form"
        st = backend.Stage(prog)
        ora = pyoracle.run_program(prog, cols, n)
        os.environ.pop("TPLX_NO_FUSED", None)
        os.environ.pop("TPLX_NO_TMA", None)
        fused_bits = st.run_host(0, cols, n).aggregate_bits()          # K3f, TMA-staged ring
        os.environ["TPLX_NO_TMA"] = "1"
        try:
            ldg_bits = st.run_host(0, cols, n).aggregate_bits()        # K3f, plain loads
        finally:
            os.environ.pop("TPLX_NO_TMA", None)
        os.environ["TPLX_NO_FUSED"] = "1"
        try:
            vm_bits = st.run_host(0, cols, n).aggregate_bits()         # K3 through the VM
        finally:
            os.environ.pop("TPLX_NO_FUSED", None)
        assert ldg_bits == fused_bits, f"program {i}: TMA vs LDG"
        assert fused_bits == vm_bits == ora.acc_tree, f"program {i}"


def test_full_block_sizes_properties(gpu):
    """At the block sizes bench.py uses: every 32,661-row cycle of the replicated Zillow input must reproduce the
    golden 577 rows (periodicity of the output), and Q6 over 50M rows must equal the oracle's tree bit for bit."""
    cols, n0 = workloads.load_zillow_fixture()
    cycles = 500
    n = cycles * n0
    big = workloads.replicate(cols, n0, n)
    prog = workloads.zillow_program()
    st = backend.Stage(prog)
    res = st.run_host(0, big, n)
    assert int(res.info.n_out_rows) == 577 * cycles and int(res.info.n_exceptions) == 0
    ora = pyoracle.run_program(prog, cols, n0)  # one cycle
    for c, (t, odata, ooffs) in enumerate(ora.columns):
        col = res.column(c)
        if t == T_STR:
            lens = np.diff(ooffs.astype(np.int64))
            assert np.array_equal(np.diff(col.offsets.astype(np.int64)), np.tile(lens, cycles)), f"col {c} lengths"
            assert col.data.tobytes() == odata.tobytes() * cycles, f"col {c} bytes"
        else:
            assert np.array_equal(col.data.view(np.int64), np.tile(odata.view(np.int64), cycles)), f"col {c}"
    res.free()
    m = 50_000_000
    lcols = workloads.gen_lineitem(m, seed=123)
    q = workloads.q6_program()
    r = backend.Stage(q).run_host(0, lcols, m)
    o = pyoracle.run_program(q, lcols, m)
    assert r.aggregate_bits() == o.acc_tree
    assert abs(ir.bits_f64(o.acc_tree[0]) - ir.bits_f64(o.acc_seq[0])) <= 1e-9 * abs(ir.bits_f64(o.acc_seq[0]))


def test_float_of_str_s2f(gpu):
    """float(str) on the device (fast_atod semantics, lazy case flags on the view) vs the oracle, incl. ValueError rows"""
    from test_float_cast import float_cases
    vals = float_cases() + ["INF", "Nan", "1E5", " 7 "]
    sc = frontend.StageCompiler([T_STR], ["s"])
    sc.add_map(lambda x: (float(x["s"]) * 2.0, float(x["s"].lower()), float(x["s"].upper()) + 1.0), 100001)
    prog = sc.finish_memory()
    col = Column.from_values(vals, T_STR)
    st, res, ora = run_both(prog, [col], len(vals))
    assert len(ora.exceptions) > 5
    assert_result_equals_oracle(res, ora, "float(str)")


def _idiom_prog(fn, with_filter=True, light=False):
    sc = frontend.StageCompiler([T_STR, T_I64], ["s", "k"])
    sc.add_with_column("r", fn, 100001)
    if with_filter:  # selective filter with heavy work behind it -> prefilter (mask kernel) + dense launch
        sc.add_filter(lambda x: x['k'] == 2, 100002)
        if light:  # nothing that materialises a copy of the (possibly very long) input string
            sc.add_with_column("t", lambda x: x['s'][0:5].replace(',', ';') + '|' + x['s'][-6:].upper() + ('%04d' % x['k']), 100003)
        else:
            sc.add_with_column("t", lambda x: x['s'].replace(',', ';') + '|' + x['s'].upper() + ('%04d' % x['k']), 100003)
        sc.add_with_column("u", lambda x: x['t'].find('BD') + int(x['s'][0:1].replace('-', '1').replace(' ', '2').replace(',', '3')
                                                                   .replace('S', '4').replace('n', '5').replace('b', '6').replace('e', '7').replace('a', '8').replace('x', '9')), 100004)
    return sc.finish_memory()


@pytest.mark.parametrize("case", ["head_len", "number_before_marker", "after_last_sep", "both_as_expr", "miss_default_one", "miss_reuse", "miss_dynamic_k"])
def test_fused_idioms_gpu_vs_oracle(gpu, case):
    """TPLX_OP_SFINDE / TPLX_OP_SRFINDK on the device (and the unfused near misses) against the oracle, with and without
    the prefilter split."""
    import idiom_udfs as U
    fn = getattr(U, case)
    n = 40_000
    cols, _ = U.make_columns(n, 3)
    for with_filter in (False, True):
        prog = _idiom_prog(fn, with_filter)
        if with_filter:
            assert prog.prefilter is not None
        st, res, ora = run_both(prog, cols, n, first_row_no=3)
        assert_result_equals_oracle(res, ora, f"{case} filter={with_filter}")


@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 64, 65, 255, 257, 8191, 8192, 8193, 100_003])
def test_mask_stage_ragged_sizes_and_modes(gpu, n):
    """K1m (mask.cuh): bitmaps + survivor list for every tail shape == oracle."""
    import idiom_udfs as U
    cols, _ = U.make_columns(n, n)
    prog = _idiom_prog(U.number_before_marker, True)
    ora = pyoracle.run_program(prog, cols, n, 11)
    res = backend.Stage(prog).run_host(0, cols, n, 11)
    assert_result_equals_oracle(res, ora, f"n={n}")


def test_mask_stage_long_strings_between_short_ones(gpu):
    _oversized_rows_check()


def _oversized_rows_check():
    """Rare very long strings (up to 12 KB) between short ones, through the prefilter and the dense launch."""
    rng = np.random.default_rng(5)
    n = 30_000
    base = ["3 bds , 2 ba", "1 bd", "x", "", "12 bds , 1 ba , 700 sqft"]
    s = [base[i] for i in rng.integers(0, len(base), n)]
    for i in rng.integers(0, n, 40):
        s[i] = ("pad," * int(rng.integers(50, 3000))) + " 7 bds , 2 ba"
    k = rng.integers(0, 4, n).astype(np.int64)
    cols = [Column.from_values(s, T_STR), Column(T_I64, k)]
    import idiom_udfs as U
    # (a stage that materialised copies of the 12 KB strings would exceed the per-row scratch arena: those rows then become
    # NORMALCASEVIOLATION rows for the resolve path by design, which is not what this test is about)
    prog = _idiom_prog(U.number_before_marker, True, light=True)
    st, res, ora = run_both(prog, cols, n)
    assert_result_equals_oracle(res, ora, "oversized rows")


def test_power_operator_gpu_vs_oracle(gpu):
    """`**` with literal exponents (multiply chains, ZeroDivisionError for 0 ** -k, guarded RAISE) on the device == oracle."""
    import power_udfs as U
    n = 30_000
    cols, _ = U.make_columns(n, 4)
    for src, _k in U.INT_CASES + U.NEG_CASES + U.FLOAT_CASES + [(m, 0) for m in U.MIXED]:
        sc = frontend.StageCompiler([T_I64, T_F64], ["a", "f"])
        sc.add_with_column("r", src, 100001)
        sc.add_filter("lambda x: x['a'] != 5", 100002)
        prog = sc.finish_memory()
        st, res, ora = run_both(prog, cols, n, first_row_no=2)
        assert_result_equals_oracle(res, ora, src)


def _vec_udf(x):
    # if-converted branches (guarded ops + phi), division that can raise inside a branch, power-of-two // and %
    a = x['a']
    if a % 4 == 1:
        r = a // (x['b'] - 2)        # ZeroDivisionError only on this branch
    elif a % 4 == 2:
        r = (a * a) // 8 - a % 16
    else:
        r = -a
    return r


@pytest.mark.parametrize("n", [0, 1, 2, 511, 512, 513, 2047, 2048, 2049, 300_001])
def test_vector_kernel_equals_scalar_kernel_and_oracle(gpu, n, monkeypatch):
    """K1v (vecvm.cuh, fixed-width stages, 128-bit loads, 8 rows per dispatch) == K1 through the scalar VM (TPLX_NO_VEC=1) == oracle:
    guarded ops, exceptions on one branch only, strength-reduced // and %, several outputs, f64 ops, ragged tails."""
    rng = np.random.default_rng(n + 1)
    a = rng.integers(-1000, 1000, n, dtype=np.int64)
    b = rng.integers(0, 5, n, dtype=np.int64)
    f = rng.normal(0, 50, n)
    sc = frontend.StageCompiler([T_I64, T_I64, T_F64], ["a", "b", "f"])
    sc.add_with_column("r", _vec_udf, 100001)
    sc.add_with_column("g", lambda x: x['f'] * 0.5 + x['a'] / 4 if x['f'] > 0.0 else abs(x['f']) % 3.0, 100002)
    sc.add_filter(lambda x: x['r'] % 3 != 0 and x['g'] < 60.0, 100003)
    sc.add_with_column("h", lambda x: (x['a'] << 2) ^ (x['b'] | 1), 100004)
    sc.add_select(["r", "g", "h", "a"], 100005)
    prog = sc.finish_memory(prefilter=False)
    cols = [Column(T_I64, a), Column(T_I64, b), Column(T_F64, f)]
    ora = pyoracle.run_program(prog, cols, n, 9)
    for env in ({}, {"TPLX_NO_VEC": "1"}):
        monkeypatch.delenv("TPLX_NO_VEC", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        res = backend.Stage(prog).run_host(0, cols, n, 9)
        assert_result_equals_oracle(res, ora, f"n={n} env={env}")
    if n > 1000:
        assert len(ora.exceptions) > 0 and 0 < ora.n_out < n


@pytest.mark.parametrize("name", ["zillow", "contains_upper", "not_contains_raw", "fixed_then_field", "field_eq_nan"])
@pytest.mark.parametrize("n", [1, 33, 50_001])
def test_string_scan_closed_form_equals_vm_and_oracle(gpu, name, n, monkeypatch):
    """K1f: the prefilter evaluated from the string-scan hint (closed form, no interpretation) == the same stage through the VM
    (TPLX_NO_SCAN=1) == oracle (which only ever runs the program): kept rows, exception rows (ValueError of int() attributed to the
    withColumn operator), row numbers."""
    import scan_udfs as U
    head = {h[0]: h[1] for h in U.HINTED}[name]
    sc = frontend.StageCompiler(U.TYPES, U.NAMES)
    head(sc)
    U.heavy_tail(sc, 100100)
    prog = sc.finish_memory()
    assert prog.prefilter is not None and ir.scan_terms(prog.prefilter.fused) is not None
    cols = U.make_columns(n, n)
    ora = pyoracle.run_program(prog, cols, n, 4)
    for env in ({}, {"TPLX_NO_SCAN": "1"}):
        monkeypatch.delenv("TPLX_NO_SCAN", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        res = backend.Stage(prog).run_host(0, cols, n, 4)
        assert_result_equals_oracle(res, ora, f"{name} n={n} env={env}")
    if n > 1000 and name in ("zillow", "fixed_then_field", "field_eq_nan"):
        assert len(ora.exceptions) > 0


def test_prefiltered_stage_without_host_round_trip(gpu, monkeypatch):
    """From the second block of a stage on, the dense launch is sized from the previous block's selectivity and reads the survivor count
    on the device (no host round trip between the two launches). Blocks with the same / far more survivors / far more exception rows
    than the estimate (retry paths), an empty block and a block without survivors must all equal the oracle; TPLX_SYNC_PREFILTER=1 (the
    round-trip path) must give the same."""
    import scan_udfs as U
    sc = frontend.StageCompiler(U.TYPES, U.NAMES)
    U._h_zillow(sc)
    U.heavy_tail(sc, 100100)
    prog = sc.finish_memory()
    rng = np.random.default_rng(77)

    def block(n, p_house, p_bad):
        f = [("x bd, y bd" if rng.random() < p_bad else U.FACTS[0]) for _ in range(n)]
        t = [("house" if rng.random() < p_house else "condo") for _ in range(n)]
        return [Column.from_values(f, T_STR), Column.from_values(t, T_STR), Column(T_I64, rng.integers(0, 9, n).astype(np.int64)),
                Column(T_F64, rng.normal(0, 1, n))]
    blocks = [(40_000, 0.02, 0.001), (40_000, 0.02, 0.001), (40_000, 0.6, 0.001), (40_000, 0.02, 0.3), (0, 0, 0), (30_000, 0.0, 0.0),
              (50_000, 0.05, 0.01)]
    data = [(block(*b), b[0]) for b in blocks]
    for env in ({}, {"TPLX_SYNC_PREFILTER": "1"}):
        monkeypatch.delenv("TPLX_SYNC_PREFILTER", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        st = backend.Stage(prog)
        for i, (cols, n) in enumerate(data):
            res = st.run_host(0, cols, n, 5)
            ora = pyoracle.run_program(prog, cols, n, 5)
            assert_result_equals_oracle(res, ora, f"block {i} env={env}")
            res.free()
        st.close()


def _keyed_with_ids(n, n_keys, seed, zipf):
    """workloads.gen_keyed, but the key ids are kept so that the expected groups come from numpy alone."""
    rng = np.random.default_rng(seed)
    ids = (np.minimum(rng.zipf(1.2, n) - 1, n_keys - 1) if zipf else rng.integers(0, n_keys, n)).astype(np.int64)
    digits = np.zeros((n, 8), dtype=np.uint8)
    digits[:, 0] = ord("k")
    x = ids.copy()
    for p in range(7, 0, -1):
        digits[:, p] = ord("0") + (x % 10)
        x //= 10
    offs = (np.arange(n + 1, dtype=np.int64) * 8).astype(np.uint32)
    return ids, Column(T_STR, digits.reshape(-1), offs)


def _ids_of_key_column(col):
    assert np.array_equal(np.diff(col.offsets.astype(np.int64)), np.full(len(col.offsets) - 1, 8))
    d = col.data.reshape(-1, 8)
    assert (d[:, 0] == ord("k")).all()
    ids = np.zeros(len(d), dtype=np.int64)
    for p in range(1, 8):
        ids = ids * 10 + (d[:, p].astype(np.int64) - ord("0"))
    return ids


@pytest.mark.parametrize("zipf", [False, True])
def test_hash_aggregate_10m_keys(gpu, zipf):
    """BASELINE config 5 at its key count (10 M distinct string keys; uniform and Zipf-distributed rows), one GPU's shard cut to
    20 M rows: i64 sums per key exact, f64 sums per key (atomics, order not fixed) within n_k * eps * sum|x| of numpy's sequential
    sums. Expected groups are computed by numpy from the generator's ids (independent of the oracle and of the device)."""
    n, n_keys = 20_000_000, 10_000_000
    ids, keycol = _keyed_with_ids(n, n_keys, 77, zipf)
    rng = np.random.default_rng(78)
    vi = rng.integers(-1000, 1000, n, dtype=np.int64)
    vf = rng.integers(-100000, 100000, n).astype(np.float64) / 64.0 + 0.1
    sc = frontend.StageCompiler([T_STR, T_I64, T_F64], ["key", "v", "f"])
    prog = sc.finish_hash(["key"], lambda a, x: (a[0] + x[1], a[1] + x[2]), lambda a, b: (a[0] + b[0], a[1] + b[1]), (0, 0.0), 100001)
    st = backend.Stage(prog)
    st.hash_reserve(0, n_keys)
    half = n // 2  # two blocks into one table, like two partitions of one task
    for lo, hi in ((0, half), (half, n)):
        cols = [Column(T_STR, keycol.data[lo * 8:hi * 8], (keycol.offsets[lo:hi + 1].astype(np.int64) - lo * 8).astype(np.uint32)),
                Column(T_I64, vi[lo:hi]), Column(T_F64, vf[lo:hi])]
        st.run_host(0, cols, hi - lo).info
    fin = st.hash_finish(0)
    got_ids = _ids_of_key_column(fin.column(0))
    present = np.unique(ids)
    assert len(got_ids) == len(present) and np.array_equal(np.sort(got_ids), present)
    want_i = np.zeros(n_keys, dtype=np.int64)
    np.add.at(want_i, ids, vi)
    assert np.array_equal(fin.column(1).data.view(np.int64), want_i[got_ids])
    want_f = np.bincount(ids, weights=vf, minlength=n_keys)
    abs_f = np.bincount(ids, weights=np.abs(vf), minlength=n_keys)
    cnt = np.bincount(ids, minlength=n_keys)
    got_f = fin.column(2).data.view(np.float64)
    bound = cnt[got_ids] * np.finfo(np.float64).eps * abs_f[got_ids] + 1e-300
    assert (np.abs(got_f - want_f[got_ids]) <= bound).all()
    st.close()
