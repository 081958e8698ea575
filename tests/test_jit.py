"""The stage specialiser (tuplex_b200/csrc/jit.inl): the op program printed as a straight-line CUDA row function and the library's own
kernel source compiled around it with NVRTC — this library's counterpart of the reference's per-stage code generation
(core/src/physical/StageBuilder.cc:602-1143, TransformStage::compile).

CPU part (no GPU): the generated text is what the program says and NVRTC turns it into an sm_90a cubin for hand-written,
workload and random programs. GPU part: with TPLX_JIT=2 (every stage specialised at its first block) results are bit-identical to
the oracle and to the interpreting kernels (TPLX_JIT=0), and the result reports that specialised kernels really ran."""
import hashlib
import os
import re

import numpy as np
import pytest

from tuplex_b200 import backend, frontend, ir, workloads as W
from oracle import pyoracle
from fuzz_udfs import COLS, TYPES, Gen, apply_ops, make_columns
from helpers import assert_result_equals_oracle

K_ROWS, K_VEC4, K_VEC2, K_AGG, K_MASK, K_WIDE4, K_RE2 = 1, 2, 3, 4, 5, 6, 10


class jit_mode:
    """TPLX_JIT is read by the library at every stage run."""

    def __init__(self, v):
        self.v = str(v)

    def __enter__(self):
        self.old = os.environ.get("TPLX_JIT")
        os.environ["TPLX_JIT"] = self.v

    def __exit__(self, *a):
        if self.old is None:
            os.environ.pop("TPLX_JIT", None)
        else:
            os.environ["TPLX_JIT"] = self.old


# ------------------------------------------------------------------------------------------------------------------
# no GPU: code generation + NVRTC
# ------------------------------------------------------------------------------------------------------------------
def test_c1_row_function_text_and_cubin():
    st = backend.Stage(W.c1_program())
    src, nb, log = st.specialise(K_VEC4)
    # x * x ; x % 2 == 0 as straight-line code on named slots: no fetch, no dispatch, constants inline
    # (% by the constant 2 is a mask on this path: the strength reduction the vector kernel's pre-decode does as well)
    assert "r1 = r0 * r0;" in src and "& 0x1ull;" in src and "floormod_i64" not in src
    assert "jit_row_fixed" in src and "out[0] = r1;" in src
    assert nb > 0, f"NVRTC produced no cubin: {log}"
    src1, nb1, log1 = st.specialise(K_ROWS)
    assert "jit_run(" in src1 and nb1 > 0, log1
    st.close()


def test_wide_tile_kinds_compile_and_other_numbers_are_rejected():
    st = backend.Stage(W.c1_program())
    for kind in (K_WIDE4, K_RE2):
        src, nb, log = st.specialise(kind)
        assert "jit_row_fixed" in src and nb > 0, log
    for kind in (0, 7, 8, 9, 11, 12):
        with pytest.raises(backend.GpuBackendError):
            st.specialise(kind)
    st.close()


def test_constant_power_of_two_divisors_are_strength_reduced():
    sc = frontend.StageCompiler([ir.T_I64], ["a"])
    sc.add_map(lambda x: (x["a"] // 8, x["a"] % 16, x["a"] // 6, x["a"] % 3, x["a"] % 1), 100001)
    st = backend.Stage(sc.finish_memory())
    src, nb, log = st.specialise(K_VEC4)
    assert nb > 0, log
    assert ">> 3);" in src and "& 0xfull;" in src and "& 0x0ull;" in src     # 2^k: shift / mask, no zero test
    assert src.count("floordiv_i64(") == 1 and src.count("floormod_i64(") == 1   # 6 and 3 keep the general form
    st.close()


def test_zillow_program_specialises():
    st = backend.Stage(W.zillow_program())
    src, nb, log = st.specialise(K_ROWS)
    assert nb > 0, log
    assert src.count("str_find(") >= 4 and "op_sreplace(" in src and "raise_exc(t, 135u" in src
    with pytest.raises(backend.GpuBackendError):  # strings: not a fixed-width stage
        st.specialise(K_VEC4)
    st.close()


def test_guarded_and_raising_ops_are_predicated():
    sc = frontend.StageCompiler([ir.T_I64, ir.T_I64], ["a", "b"])
    sc.add_map(lambda x: x["a"] // x["b"] if x["b"] != 0 else -1, 100001)
    st = backend.Stage(sc.finish_memory())
    src, nb, log = st.specialise(K_VEC4)
    assert nb > 0, log
    # the division sits under its guard and raises ZeroDivisionError (136) only on the executed path
    lines = [l for l in src.splitlines() if "IFLOORDIV" in l]
    assert lines and all(l.split("*/")[1].strip().startswith("if (r") for l in lines), src
    assert "136u" in src
    st.close()


@pytest.mark.parametrize("seed", range(3))
def test_random_pipelines_compile(seed):
    g = Gen(7000 + seed)
    done = 0
    for _ in range(12):
        ops = g.pipeline()
        sc = frontend.StageCompiler(TYPES, COLS)
        try:
            apply_ops(sc, ops)
            prog = sc.finish_memory(prefilter=False)
        except frontend.UnsupportedUDF:
            continue
        st = backend.Stage(prog)
        src, nb, log = st.specialise(K_ROWS)
        assert nb > 0, f"{ops}\n{src}\n{log}"
        if st.vec_plan() is not None:
            src, nb, log = st.specialise(K_VEC4)
            assert nb > 0, f"{ops}\n{src}\n{log}"
        st.close()
        done += 1
        if done >= 4:
            break
    assert done >= 2


# ------------------------------------------------------------------------------------------------------------------
# GPU: specialised kernels vs oracle vs interpreting kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 2047, 2048, 100_003, 1_000_001])
def test_c1_specialised_vector_kernel(gpu, n):
    x = np.arange(1, n + 1, dtype=np.int64) * 3 - 7
    cols = [backend.Column(ir.T_I64, x)]
    prog = W.c1_program()
    ora = pyoracle.run_program(prog, cols, n)
    for mode in (2, 0):
        with jit_mode(mode):
            st = backend.Stage(prog)
            res = st.run_host(0, cols, n)
            assert_result_equals_oracle(res, ora, f"C1 n={n} TPLX_JIT={mode}")
            if n:
                assert (int(res.info.specialised_launches) > 0) == (mode == 2), "specialised kernel did not run" if mode else "interpreter expected"
            res.free()
            st.close()


@pytest.mark.gpu
def test_fixed_width_exceptions_and_branches(gpu):
    n = 300_001
    rng = np.random.default_rng(5)
    a = rng.integers(-1000, 1000, n)
    b = rng.integers(-3, 4, n)  # zeros: ZeroDivisionError rows
    f = rng.integers(-50, 50, n) / 4.0
    cols = [backend.Column(ir.T_I64, a), backend.Column(ir.T_I64, b), backend.Column(ir.T_F64, f)]
    sc = frontend.StageCompiler([ir.T_I64, ir.T_I64, ir.T_F64], ["a", "b", "f"])
    sc.add_with_column("q", lambda x: x["a"] // x["b"], 100001)
    sc.add_with_column("m", lambda x: x["a"] % x["b"] if x["a"] > 0 else x["a"] * 2, 100002)
    sc.add_filter(lambda x: x["q"] != 3, 100003)
    sc.add_with_column("g", lambda x: x["f"] / (x["f"] - 2.5), 100004)
    sc.add_map(lambda x: (x["q"], x["m"], x["g"], x["a"] + 1), 100005)
    prog = sc.finish_memory(prefilter=False)
    ora = pyoracle.run_program(prog, cols, n, first_row_no=11)
    assert len(ora.exceptions) > 100
    for mode in (2, 0):
        with jit_mode(mode):
            st = backend.Stage(prog)
            res = st.run_host(0, cols, n, first_row_no=11)
            assert_result_equals_oracle(res, ora, f"TPLX_JIT={mode}")
            assert (int(res.info.specialised_launches) > 0) == (mode == 2)
            res.free()
            st.close()


@pytest.mark.gpu
def test_strength_reduced_divisions_on_negative_values(gpu):
    """x // 2^k and x % 2^k as shift / mask must keep Python's floor semantics for negative x (specialised == interpreted == oracle)."""
    n = 200_003
    rng = np.random.default_rng(17)
    a = rng.integers(-(1 << 40), 1 << 40, n)
    a[:4] = [-(1 << 63), (1 << 63) - 1, -1, 0]
    cols = [backend.Column(ir.T_I64, a)]
    sc = frontend.StageCompiler([ir.T_I64], ["a"])
    sc.add_map(lambda x: (x["a"] // 8, x["a"] % 16, x["a"] // 1, x["a"] % 1, x["a"] // 4096, x["a"] % 2), 100001)
    sc.add_filter(lambda a, b, c, d, e, f: f == 1 or b > 3, 100002)
    prog = sc.finish_memory(prefilter=False)
    ora = pyoracle.run_program(prog, cols, n)
    for mode in (2, 0):
        with jit_mode(mode):
            st = backend.Stage(prog)
            res = st.run_host(0, cols, n)
            assert_result_equals_oracle(res, ora, f"TPLX_JIT={mode}")
            res.free()
            st.close()
    want = [(int(v) // 8, int(v) % 16, int(v), 0, int(v) // 4096, int(v) % 2) for v in a.tolist()]
    want = [w for w in want if w[5] == 1 or w[1] > 3]
    assert list(zip(*[ora.values(c) for c in range(6)])) == want  # and the oracle is CPython's floor semantics


@pytest.mark.gpu
def test_zillow_specialised_matches_golden_md5(gpu):
    src, n0 = W.load_zillow_fixture()
    n = 5 * n0 + 1234
    cols = W.replicate(src, n0, n)
    prog = W.zillow_program()
    ora = pyoracle.run_program(prog, cols, n)
    outs = {}
    for mode in (2, 0):
        with jit_mode(mode):
            st = backend.Stage(prog)
            res = st.run_host(0, cols, n)
            assert_result_equals_oracle(res, ora, f"zillow TPLX_JIT={mode}")
            outs[mode] = int(res.info.specialised_launches)
            res.free()
            st.close()
    assert outs[2] > 0 and outs[0] == 0
    # and the golden file of the reference's own zillow.cpp / runpython.py, through the specialised kernels
    with jit_mode(2):
        st = backend.Stage(prog)
        res = st.run_host(0, src, n0)
        assert int(res.info.specialised_launches) > 0
        txt = W.rows_to_csv([c.to_values() for c in res.columns()], W.ZILLOW_OUT)
        assert hashlib.md5(txt).hexdigest() == "4d5ca0263b1a5058341a369116dee83a"
        res.free()
        st.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_random_pipelines_specialised_match_oracle(gpu, seed):
    g = Gen(4200 + seed)
    n = 30_000 + 41 * seed
    cols, _ = make_columns(n, seed)
    compared = 0
    with jit_mode(2):
        for trial in range(12):
            ops = g.pipeline()
            progs = []
            for pre in (True, False):
                sc = frontend.StageCompiler(TYPES, COLS)
                try:
                    apply_ops(sc, ops)
                    progs.append(sc.finish_memory(prefilter=pre))
                except frontend.UnsupportedUDF:
                    progs = []
                    break
            if not progs:
                continue
            ora = pyoracle.run_program(progs[1], cols, n, first_row_no=seed)
            for prog in progs if progs[0].prefilter is not None else progs[1:]:
                st = backend.Stage(prog)
                res = st.run_host(0, cols, n, first_row_no=seed)
                assert_result_equals_oracle(res, ora, f"seed {seed} trial {trial} prefilter={prog.prefilter is not None}: {ops}")
                if prog.prefilter is None and ora.n_out + len(ora.exceptions) > 0:
                    assert int(res.info.specialised_launches) > 0
                res.free()
                st.close()
            compared += 1
            if compared >= 5:
                break
    assert compared >= 3


@pytest.mark.gpu
def test_tiered_execution_background_compile(gpu):
    """Default policy: the first blocks of a hot stage run on the interpreting kernel while NVRTC compiles on a background thread;
    later blocks run the specialised kernel. Every block gives the same result."""
    import time
    n = 200_000
    x = np.arange(1, n + 1, dtype=np.int64)
    cols = [backend.Column(ir.T_I64, x)]
    prog = W.c1_program()
    ora = pyoracle.run_program(prog, cols, n)
    old = {k: os.environ.get(k) for k in ("TPLX_JIT", "TPLX_JIT_MIN_ROWS", "TPLX_JIT_SYNC")}
    os.environ.update(TPLX_JIT="1", TPLX_JIT_MIN_ROWS="1000", TPLX_JIT_SYNC="0")
    try:
        st = backend.Stage(prog)
        seen = []
        t0 = time.time()
        while time.time() - t0 < 60:
            res = st.run_host(0, cols, n)
            assert_result_equals_oracle(res, ora, "tiered")
            seen.append(int(res.info.specialised_launches))
            res.free()
            if seen[-1]:
                break
            time.sleep(0.05)
        assert seen[-1] > 0, "the specialised kernel never took over"
        assert seen[0] == 0, "the first block waited for the compiler"
        st.close()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# Program shapes and the specialised fixed-width kernel each one selects (run_rows_vec): at most 16 instructions -> K1r; else K1w
# when the live-out slots of four 2048-row sub-batches fit 74 KB of shared memory (one slot); else K1v with J = 4 when they fit 56 KB
# (two slots), else with J = 2 within 100 KB (three to eleven slots). name: (more than 16 instructions, final map, kind)
WIDE_SHAPES = {
    "re2": (False, None, K_RE2),
    "re2_2out": (False, lambda x: (x, x * 2 + 1), K_RE2),
    "wide4": (True, None, K_WIDE4),
    "vec4": (True, lambda x: (x, x * 2 + 1), K_VEC4),
    "vec2": (True, lambda x: (x, x * 2 + 1, x - 5), K_VEC2),
    "vec2_11out": (True, lambda x: (x, x + 1, x + 2, x + 3, x + 4, x + 5, x + 6, x + 7, x + 8, x + 9, x + 10), K_VEC2),
}


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 8191, 8192, 8193, 16385, 100_003, 3_000_001])
@pytest.mark.parametrize("shape", list(WIDE_SHAPES))
def test_wide_tile_kernels_with_exceptions(gpu, n, shape, monkeypatch, capfd):
    """The specialised fixed-width kernels vs the oracle, each selected by the shape of its program — K1r (nothing staged, the tile is
    evaluated again from L2 once its offset is known; 2 sub-batches of 2048 rows per ticket, two tiles in flight per CTA), K1w (live-out
    slots of 4 sub-batches staged in shared memory), K1v with J = 4 and J = 2 — on ragged tiles, with ZeroDivisionError rows and a filter.
    The trace names the kind that was loaded."""
    long, final_map, kind = WIDE_SHAPES[shape]
    rng = np.random.default_rng(n)
    a = rng.integers(-10_000, 10_000, n)
    cols = [backend.Column(ir.T_I64, a)]
    sc = frontend.StageCompiler([ir.T_I64], ["a"])
    sc.add_map(lambda x: x // (x % 7), 100001)       # x % 7 == 0 raises
    sc.add_filter(lambda x: x % 3 != 1, 100002)
    if long:
        sc.add_map(lambda x: ((x * 3 + 1) ^ (x >> 2)) + ((x * 5 - 7) & 1023) - (x | 96) + (x << 1), 100003)
    if final_map is not None:
        sc.add_map(final_map, 100004)
    prog = sc.finish_memory(prefilter=False)
    assert (len(prog.instrs) > 16) == long
    ora = pyoracle.run_program(prog, cols, n, first_row_no=5)
    monkeypatch.setenv("TPLX_TRACE", "1")
    capfd.readouterr()
    with jit_mode(2):
        st = backend.Stage(prog)
        res = st.run_host(0, cols, n, first_row_no=5)
        assert_result_equals_oracle(res, ora, f"n={n} shape={shape}")
        assert int(res.info.specialised_launches) > 0
        res.free()
        st.close()
    assert re.findall(r"specialiser: kind (\d+) loaded", capfd.readouterr().err) == [str(kind)]
