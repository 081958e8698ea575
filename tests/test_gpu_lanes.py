"""Blocks of one stage in flight from several threads, the way bench.py runs them (`ThreadPoolExecutor(max_workers=3).map` over a
stage's blocks): every call enters tplx_gpu_stage_run / tplx_gpu_stage_run_host together with two others, so one runs on the GPU's
primary execution lane, the next on its second lane (`Device::alt`, own streams, scratch and page-locked count buffer) and the third
waits for a lane. The lanes share the stage's run-time estimates (string bytes and exception rows per row, the prefilter's survivor
ratio), its `prefilter_enabled` switch, the lazily built K1v program and the specialiser's state, so one lane's block sizes the
other lane's launches.

Every job is checked bit for bit against two references: the CPU oracle on the same rows with the same first row number, and the
same block run alone on a fresh Stage. Every block differs from every other block in content and first row number, so a result
handed to the wrong caller, counts read from the other lane's buffer, or rows numbered from another block's base fail the
comparison. Each case also asserts which lanes ran its jobs (tplx_result_info.lane), so that it cannot pass without the second
lane; hash stages keep to the primary lane. A line per case, printed with -rA, shows the lanes, the retried blocks and the
interpreted / specialised split."""
import contextlib
import os
import re
import threading
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import pytest

import scan_udfs as U
from helpers import assert_result_equals_oracle
from oracle import pyoracle
from tuplex_b200 import backend, frontend, ir, workloads
from tuplex_b200.backend import Column, pack_valid
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR

pytestmark = pytest.mark.gpu

K_ROWS = 1      # stage specialiser kind of the row kernel K1 (include/tplx_gpu.h, tplx_gpu_stage_specialise)
MASK_LAUNCHES = 4  # K1m / K1f: mask kernel, count, scan, expand


# ---- harness ---------------------------------------------------------------------------------------------------------------
@dataclass
class Run:
    res: backend.Result
    lane: int
    launches: int
    specialised: int
    zero_copy: int = 0


def _runs(call, jobs, workers):
    """call(job) for every job on `workers` threads, in rounds of `workers` jobs that pass a barrier together right before the call."""
    out: List[Optional[Run]] = [None] * len(jobs)
    with ThreadPoolExecutor(max_workers=workers) as pool:
        for lo in range(0, len(jobs), workers):
            idx = list(range(lo, min(lo + workers, len(jobs))))
            bar = threading.Barrier(len(idx))

            def one(i, bar=bar):
                bar.wait(timeout=120)
                res = call(jobs[i])
                inf = res.info
                return Run(res, int(inf.lane), int(inf.kernel_launches), int(inf.specialised_launches), int(inf.zero_copy_cols))
            for i, r in zip(idx, pool.map(one, idx)):
                out[i] = r
    return out


def run_concurrently(stage, jobs, workers=3):
    """(block, first_row_no) jobs through stage.run, `workers` calls at a time (bench.py step_resident)."""
    return _runs(lambda j: stage.run(j[0], j[1]), jobs, workers)


def run_host_concurrently(stage, jobs, workers=3):
    """(host columns, n_rows, first_row_no) jobs through stage.run_host, `workers` calls at a time (bench.py step_e2e)."""
    return _runs(lambda j: stage.run_host(0, j[0], j[1], j[2]), jobs, workers)


def pinned(arr: np.ndarray):
    """Copy a numpy array into page-locked host memory (torch is the allocator only); returns the view and its owner."""
    import torch
    t = torch.empty(arr.shape, dtype=torch.from_numpy(arr[:0]).dtype, pin_memory=True)
    out = t.numpy()
    out[...] = arr
    return out, t


def pinned_columns(cols, keep):
    out = []
    for c in cols:
        d, k = pinned(c.data)
        keep.append(k)
        o = None
        if c.offsets is not None:
            o, k = pinned(c.offsets)
            keep.append(k)
        out.append(Column(c.type, d, o, c.valid))
    return out


@dataclass
class Snap:
    """Everything a result hands back, fetched to the host."""
    n_out: int
    cols: list
    valid: list
    exc: np.ndarray
    agg: Optional[list] = None
    launches: int = 0


def snapshot(res: backend.Result, aggregate=False) -> Snap:
    inf = res.info
    if aggregate:
        return Snap(int(inf.n_out_rows), [], [], res.exceptions(), res.aggregate_bits(), int(inf.kernel_launches))
    cols = res.columns()
    return Snap(int(inf.n_out_rows), [(c.type, c.data.tobytes(), None if c.offsets is None else c.offsets.tobytes()) for c in cols],
                [None if c.valid is None else c.valid.tobytes() for c in cols], res.exceptions(), None, int(inf.kernel_launches))


def assert_same(got: Snap, want: Snap, what):
    assert got.n_out == want.n_out, f"{what}: {got.n_out} rows, alone {want.n_out}"
    assert got.agg == want.agg, f"{what}: aggregate differs from the block run alone"
    assert len(got.cols) == len(want.cols)
    for c, (g, w) in enumerate(zip(got.cols, want.cols)):
        assert g == w, f"{what}: column {c} differs from the block run alone"
    assert got.valid == want.valid, f"{what}: validity words differ from the block run alone"
    for f in ("row", "row_no", "code", "op_id"):
        assert np.array_equal(got.exc[f], want.exc[f]), f"{what}: exception field {f} differs from the block run alone"


def alone(prog, block, first_row_no, aggregate=False):
    st = backend.Stage(prog)
    res = st.run(block, first_row_no)
    snap = snapshot(res, aggregate)
    res.free()
    st.close()
    return snap


@contextlib.contextmanager
def environ(**kv):
    """Environment variables for the references that module-scoped fixtures compute (monkeypatch is function-scoped)."""
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def report(case, runs, retried=(), extra=""):
    """retried: blocks that took more launches than alone, or that retried by construction"""
    lanes = sorted({r.lane for r in runs})
    spec = sum(r.specialised > 0 for r in runs)
    print(f"[lanes] {case}: {len(runs)} jobs, lanes {lanes} (lane 1: {sum(r.lane == 1 for r in runs)} jobs), retried {list(retried)}, "
          f"{len(runs) - spec} interpreted / {spec} specialised {extra}")


def assert_both_lanes(case, runs):
    lanes = {r.lane for r in runs}
    assert lanes == {0, 1}, f"{case}: jobs ran on lanes {sorted(lanes)}; concurrent calls must use both execution lanes"


def str_col(vocab, idx, valid=None) -> Column:
    enc = [v.encode() for v in vocab]
    lens = np.array([len(e) for e in enc], np.int64)[idx]
    offs = np.zeros(len(idx) + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    data = np.frombuffer(b"".join(map(enc.__getitem__, idx.tolist())), np.uint8).copy() if len(idx) else np.zeros(0, np.uint8)
    return Column(T_STR, data, offs.astype(np.uint32), valid)


# ---- (a) Zillow Z1, device-resident ------------------------------------------------------------------------------------------
# (rotation of the fixture, rows): lengths around 10^6 rows, one not a multiple of 32, one under 2^16 rows
ZILLOW_BLOCKS = [(0, 1_000_000), (1234, 917_777), (5_000, 40_001), (17_000, 1_100_032), (30_001, 654_321), (9_999, 800_003),
                 (22_222, 333_335), (31_000, 1_000_017)]


def zillow_block(rot, n):
    cols, n0 = workloads.load_zillow_fixture()
    r = workloads.replicate(cols, n0, n0 + rot + n)
    return [c.slice(rot, rot + n) for c in r]


@pytest.fixture(scope="module")
def zillow_case(gpu):
    prog = workloads.zillow_program()
    golden = workloads.zillow_golden_csv().decode().split("\n")[1:-1]
    blocks = []
    with environ(TPLX_JIT="0"):
        for i, (rot, n) in enumerate(ZILLOW_BLOCKS):
            cols = zillow_block(rot, n)
            first = 1000 * i + 7
            blk = backend.Block.upload(0, cols, n)
            ora = pyoracle.run_program(prog, cols, n, first)
            blocks.append((blk, first, ora, alone(prog, blk, first)))
    yield prog, golden, blocks
    for b in blocks:
        b[0].free()


def assert_golden_cycles(res, golden, what):
    """The rows of a rotated fixture are the golden rows from some position on, cyclically: every full cycle the block holds
    reproduces the golden output."""
    vals = [c.to_values() for c in res.columns()]
    lines = workloads.rows_to_csv(vals, None).decode().split("\n")[:-1]
    assert len(lines) > 0, what
    m = len(golden)
    starts = [j for j in range(m) if golden[j] == lines[0]]
    ok = any(all(lines[t] == golden[(j + t) % m] for t in range(len(lines))) for j in starts)
    assert ok, f"{what}: output rows are not the golden rows of the cycles the block holds"


@pytest.mark.parametrize("mode", ["interpreted", "tiered"])
def test_zillow_blocks_on_both_lanes(zillow_case, mode, monkeypatch):
    """(a) The bench's stage over distinct blocks, three calls at a time. `tiered`: TPLX_JIT=1 with a lowered threshold and no
    TPLX_JIT_SYNC, so the first rounds start the background compile and run interpreted; the compile is awaited before the last
    round, whose blocks run specialised while blocks of the same stage ran interpreted before them."""
    prog, golden, blocks = zillow_case
    monkeypatch.delenv("TPLX_JIT_SYNC", raising=False)
    if mode == "interpreted":
        monkeypatch.setenv("TPLX_JIT", "0")
    else:
        monkeypatch.setenv("TPLX_JIT", "1")
        monkeypatch.setenv("TPLX_JIT_MIN_ROWS", str(1 << 16))
    st = backend.Stage(prog)
    jobs = [(b[0], b[1]) for b in blocks]
    if mode == "interpreted":
        runs = run_concurrently(st, jobs)
        nvrtc = False
    else:
        runs = run_concurrently(st, jobs[:6])
        nvrtc = st.specialise(K_ROWS, compile=True)[1] > 0  # waits for the background compile the first rounds started
        runs += run_concurrently(st, jobs[6:])
    for i, (run, (blk, first, ora, ref)) in enumerate(zip(runs, blocks)):
        what = f"zillow {mode} block {i} (lane {run.lane}, {'specialised' if run.specialised else 'interpreted'})"
        assert_result_equals_oracle(run.res, ora, what)
        assert_same(snapshot(run.res), ref, what)
        assert_golden_cycles(run.res, golden, what)
        if mode == "interpreted":
            assert run.specialised == 0, what
        run.res.free()
    report(f"zillow {mode}", runs)
    if nvrtc:
        assert any(r.specialised for r in runs), "NVRTC is present but no block ran the specialised kernel"
        assert any(r.specialised == 0 for r in runs[:3]), "the first round must run before the compile has finished"
    assert_both_lanes(f"zillow {mode}", runs)
    st.close()


# ---- (b) estimates shared between lanes ---------------------------------------------------------------------------------------
BAD_FACTS = "x bd, y bd"   # bedrooms(): int('x') raises in the prefilter
GOOD_FACTS = "3 bd"        # 3 bedrooms


def scan_program():
    """scan_udfs' Zillow head (string-scan prefilter) + heavy_tail + a column that raises ZeroDivisionError where k == 3, so the dense
    launch writes exception records too."""
    sc = frontend.StageCompiler(U.TYPES, U.NAMES)
    U._h_zillow(sc)
    U.heavy_tail(sc, 100100)
    sc.add_with_column("z4", lambda x: 1000 // (x['k'] - 3), 100103)
    prog = sc.finish_memory()
    assert prog.prefilter is not None and ir.scan_terms(prog.prefilter.fused) is not None
    return prog


def scan_block(n, p_surv, p_pexc, p_dexc, seed, title_len=0):
    """p_surv: rows whose title holds 'house' (survivors), p_pexc: rows whose facts make the prefilter raise, p_dexc: rows with k == 3
    (ZeroDivisionError behind the prefilter); title_len pads every title to that many bytes (string bytes per row; the stage's
    per-row string arena holds the heavy tail's temporaries of titles up to about 55 bytes)."""
    rng = np.random.default_rng(seed)
    pad = "x" * max(0, title_len - 5)
    titles = ["House" + pad, "condo" + pad]
    t = (rng.random(n) >= p_surv).astype(np.int64)
    f = (rng.random(n) < p_pexc).astype(np.int64)
    k = rng.integers(4, 12, n).astype(np.int64)
    k[rng.random(n) < p_dexc] = 3
    return [str_col([GOOD_FACTS, BAD_FACTS], f), str_col(titles, t), Column(T_I64, k), Column(T_F64, rng.normal(0, 3, n))]


# name: (rows, survivor share, prefilter exception share, dense exception share, title bytes)
SCAN_WARM = ("warm", (100_000, 0.02, 0.001, 0.0, 0))
# Round 1 runs in rounds of three in this order: L and E are sized from the warm-up block, B1 or each other (survivor ratio
# <= 0.06), S from a block of the second round.
SCAN_ROUND1 = [
    ("B1", (1_000_000, 0.02, 0.001, 0.001, 0)),
    ("L", (1_000_000, 0.06, 0.001, 0.0, 55)),    # 11x the title bytes per survivor: string capacity retry (flag 2)
    ("E", (1_000_000, 0.03, 0.001, 0.9, 0)),     # most survivors raise behind the prefilter: exception capacity retry (flag 4)
    ("P", (1_000_000, 0.01, 0.3, 0.0, 0)),       # 30 % prefilter exceptions: re-expanded with the exact capacity
    ("empty", (0, 0.0, 0.0, 0.0, 0)),
    ("none", (500_000, 0.0, 0.0, 0.0, 0)),       # no survivor at all
    ("S", (1_000_000, 0.3, 0.001, 0.001, 0)),    # more survivors than any other block's ratio sizes for: survivor retry (flag 8)
    ("B2", (700_001, 0.05, 0.01, 0.01, 0)),
]
SCAN_ROUND2 = [  # N is not selective and >= 2^16 rows: it switches the prefilter off while the others are in flight
    ("N", (200_000, 0.9, 0.001, 0.01, 0)),
    ("B3", (600_000, 0.02, 0.002, 0.02, 0)),
    ("B4", (400_003, 0.04, 0.001, 0.0, 0)),
    ("B5", (900_000, 0.01, 0.01, 0.05, 0)),
    ("B6", (333_333, 0.03, 0.0, 0.0, 0)),
]


@pytest.fixture(scope="module")
def scan_case(gpu):
    prog = scan_program()
    blocks = {}
    with environ(TPLX_JIT="0"):
        for i, (name, spec) in enumerate([SCAN_WARM] + SCAN_ROUND1 + SCAN_ROUND2):
            n = spec[0]
            cols = scan_block(*spec[:4], seed=100 + i, title_len=spec[4])
            first = 10_000 * i + 3
            blk = backend.Block.upload(0, cols, n)
            blocks[name] = dict(cols=cols, n=n, first=first, blk=blk, ora=pyoracle.run_program(prog, cols, n, first),
                                ref=alone(prog, blk, first))

    def survivors(v):  # rows the prefilter keeps: output rows + the dense launch's exception rows
        return v["ora"].n_out + int((v["ora"].exceptions["op_id"] == 100103).sum())
    # the survivor retry is there by construction: S has more survivors than the dense launch is sized for from any other block
    ratios = {k: survivors(v) / v["n"] for k, v in blocks.items() if v["n"] and k not in ("S", "N")}
    s = blocks["S"]
    assert survivors(s) > max(ratios.values()) * 1.3 * s["n"] + 65536
    assert survivors(blocks["N"]) * 2 > blocks["N"]["n"] >= 1 << 16
    assert all(survivors(blocks[k]) < 65536 for k in ratios)  # only S outgrows the dense launch's minimum capacity
    yield prog, blocks
    for v in blocks.values():
        v["blk"].free()


@pytest.mark.parametrize("scan", ["K1f", "K1m"])
def test_prefiltered_estimates_shared_between_lanes(scan_case, scan, monkeypatch, capfd):
    """(b) Blocks whose survivor ratio, exception rates and output string bytes per row differ 10-100x, three at a time on one
    stage: each block is sized from whichever block finished before it, on either lane. The retries must give the same rows as the
    block alone and the oracle. K1f = the prefilter's closed form, K1m = the interpreted mask kernel (TPLX_NO_SCAN=1)."""
    prog, blocks = scan_case
    monkeypatch.setenv("TPLX_JIT", "0")
    monkeypatch.delenv("TPLX_SYNC_PREFILTER", raising=False)
    if scan == "K1m":
        monkeypatch.setenv("TPLX_NO_SCAN", "1")
    else:
        monkeypatch.delenv("TPLX_NO_SCAN", raising=False)
    st = backend.Stage(prog)
    w = blocks["warm"]
    st.run(w["blk"], w["first"]).free()  # every later block takes the path without a host round trip (sized from estimates)
    capfd.readouterr()
    monkeypatch.setenv("TPLX_TRACE", "1")
    names1 = [n for n, _ in SCAN_ROUND1]
    runs1 = run_concurrently(st, [(blocks[n]["blk"], blocks[n]["first"]) for n in names1])
    monkeypatch.delenv("TPLX_TRACE")
    trace = capfd.readouterr().err
    names2 = [n for n, _ in SCAN_ROUND2]
    runs2 = run_concurrently(st, [(blocks[n]["blk"], blocks[n]["first"]) for n in names2])
    retried = []
    for name, run in zip(names1 + names2, runs1 + runs2):
        b = blocks[name]
        what = f"{scan} block {name} (lane {run.lane}, {run.launches} launches, alone {b['ref'].launches})"
        assert_result_equals_oracle(run.res, b["ora"], what)
        assert_same(snapshot(run.res), b["ref"], what)
        if run.launches > b["ref"].launches:
            retried.append(name)
        run.res.free()
    by = dict(zip(names1, runs1))
    # string bytes: sized from short-title blocks, L needs a second attempt that it does not need alone (sized from its input bytes)
    assert by["L"].launches > blocks["L"]["ref"].launches, "L's dense launch must retry for string bytes"
    # exceptions behind the prefilter: E needs the second attempt of the dense launch (alone too: its first capacity is a floor)
    assert by["E"].launches == MASK_LAUNCHES + 2, "E's dense launch must retry for exception records"
    # survivors: the count is reset by the exactly sized second dense launch, so the trace shows it: one dense launch per block
    # with rows, and S's second one
    dense = len(re.findall(r"\[tplx\] rows kernel", trace))
    assert dense == sum(1 for n in names1 if blocks[n]["n"]) + 1, f"{dense} dense launches in round 1:\n{trace[-4000:]}"
    assert st_prefilter_off(st, blocks)
    report(f"prefiltered {scan}", runs1 + runs2, retried + ["S (survivors)"], f"; {dense} dense launches in round 1")
    assert_both_lanes(f"prefiltered {scan} round 1", runs1)
    assert_both_lanes(f"prefiltered {scan}", runs1 + runs2)
    st.close()


def st_prefilter_off(st, blocks):
    """After N the stage runs without its prefilter: a block then takes one launch, no mask launches."""
    b = blocks["B6"]
    res = st.run(b["blk"], b["first"])
    assert_result_equals_oracle(res, b["ora"], "B6 after the prefilter was switched off")
    launches = int(res.info.kernel_launches)
    res.free()
    assert launches < MASK_LAUNCHES, f"the non-selective block must switch the prefilter off ({launches} launches)"
    return True


# ---- (c) K1v and Option columns ----------------------------------------------------------------------------------------------
def _vec_udf(x):
    a = x['a']
    if a % 4 == 1:
        r = a // (x['b'] - 2)
    elif a % 4 == 2:
        r = (a * a) // 8 - a % 16
    else:
        r = -a
    return r


def vec_program():
    sc = frontend.StageCompiler([T_I64, T_I64, T_F64], ["a", "b", "f"])
    sc.add_with_column("r", _vec_udf, 100001)
    sc.add_with_column("g", lambda x: x['f'] * 0.5 + x['a'] / 4 if x['f'] > 0.0 else abs(x['f']) % 3.0, 100002)
    sc.add_filter(lambda x: x['r'] % 3 != 0 and x['g'] < 60.0, 100003)
    sc.add_with_column("h", lambda x: (x['a'] << 2) ^ (x['b'] | 1), 100004)
    sc.add_select(["r", "g", "h", "a"], 100005)
    prog = sc.finish_memory(prefilter=False)
    assert backend.Stage(prog).vec_plan() is not None
    return prog


def test_vector_kernel_program_built_on_both_lanes(gpu, monkeypatch):
    """(c) A fixed-width stage (K1v), three blocks at once on a fresh Stage, three times over: the first calls on both lanes build
    the K1v program lazily at the same time."""
    monkeypatch.setenv("TPLX_JIT", "0")
    prog = vec_program()
    runs = []
    for rep in range(3):
        jobs, refs = [], []
        for j, n in enumerate((1_000_003, 750_000, 1_200_001)):
            rng = np.random.default_rng(10 * rep + j)
            cols = [Column(T_I64, rng.integers(-1000, 1000, n, dtype=np.int64)), Column(T_I64, rng.integers(0, 5, n, dtype=np.int64)),
                    Column(T_F64, rng.normal(0, 50, n))]
            first = 100 * rep + 11 * j
            blk = backend.Block.upload(0, cols, n)
            jobs.append((blk, first))
            refs.append((pyoracle.run_program(prog, cols, n, first), alone(prog, blk, first)))
        st = backend.Stage(prog)
        got = run_concurrently(st, jobs)
        for j, (run, (ora, ref)) in enumerate(zip(got, refs)):
            what = f"K1v repetition {rep} block {j} (lane {run.lane})"
            assert_result_equals_oracle(run.res, ora, what)
            assert_same(snapshot(run.res), ref, what)
            assert len(ora.exceptions) > 0, what
            run.res.free()
        st.close()
        for b, _ in jobs:
            b.free()
        runs += got
    report("K1v", runs)
    assert_both_lanes("K1v", runs)


OPT_NAMES = ["a", "b", "s"]
OPT_TYPES = [T_I64, T_I64, T_STR]


def _opt_udf(x):
    return (x['a'], x['s'], x['a'] * 2 if x['a'] is not None else x['b'])


def option_block(n, seed):
    rng = np.random.default_rng(seed)
    pa = rng.random(n) >= 0.3
    ps = rng.random(n) >= 0.2
    a = np.where(pa, rng.integers(-50, 50, n), 0).astype(np.int64)
    s = np.where(ps, rng.integers(0, 5, n), 0)
    return [Column(T_I64, a, None, pack_valid(pa)), Column(T_I64, rng.integers(0, 100, n).astype(np.int64)),
            str_col(["", "abc", "Banana", "xyz", "A"], s, pack_valid(ps))]


def expanded(cols, prog):
    """The program's input: physical columns + one `is None` companion per Option column (what the executor builds)."""
    out = [Column(c.type, c.data, c.offsets, c.valid) for c in cols]
    for j in sorted(prog.null_of):
        pres = cols[prog.null_of[j]].present()
        out.append(Column(T_BOOL, (~pres).astype(np.int64) if pres is not None else np.zeros(len(cols[0]), np.int64)))
    return out


def oracle_validity(prog, ora):
    """Validity words per visible output column from the oracle's `is None` companion columns (None: the column has none)."""
    n_vis = len(prog.out_cols) - prog.hidden_out_cols
    valid = [None] * n_vis
    for k, nof in enumerate(prog.out_null_of):
        if nof:
            isnull = ora.columns[k][1].astype(bool)
            valid[nof - 1] = pack_valid(~isnull).tobytes()
    return valid


def test_option_columns_on_both_lanes(gpu, monkeypatch):
    """(c) Option[i64] / Option[str] inputs and Option outputs: the `is None` companions are expanded from the blocks' validity
    words and the outputs' companions packed into validity words on whichever lane ran the block; words compared exactly."""
    monkeypatch.setenv("TPLX_JIT", "0")
    sc = frontend.StageCompiler(OPT_TYPES, OPT_NAMES, [0, 2])
    sc.add_map(_opt_udf, 100001)
    prog = sc.finish_memory()
    assert prog.null_of and any(prog.out_null_of)
    jobs, refs = [], []
    for j, n in enumerate((1_000_001, 640_000, 900_017, 64_000, 1_100_000, 777_777)):
        cols = option_block(n, 500 + j)
        first = 37 * j + 1
        blk = backend.Block.upload(0, cols, n)
        ora = pyoracle.run_program(prog, expanded(cols, prog), n, first)
        jobs.append((blk, first))
        refs.append((ora, alone(prog, blk, first)))
    st = backend.Stage(prog)
    runs = run_concurrently(st, jobs)
    n_vis = len(prog.out_cols) - prog.hidden_out_cols
    for j, (run, (ora, ref)) in enumerate(zip(runs, refs)):
        what = f"Option block {j} (lane {run.lane})"
        snap = snapshot(run.res)
        assert_same(snap, ref, what)
        assert snap.n_out == ora.n_out, what
        valid = oracle_validity(prog, ora)
        assert snap.valid == valid, f"{what}: validity words differ from the oracle"
        for c in range(n_vis):  # values of the rows that hold one (a None row's placeholder is not a value)
            want = ora.values(c)
            if valid[c] is not None:
                pres = backend.unpack_valid(np.frombuffer(valid[c], np.uint32), ora.n_out)
                want = [v if p else None for v, p in zip(want, pres.tolist())]
            assert run.res.column(c).to_values() == want, f"{what}: column {c} differs from the oracle"
        for f in ("row", "row_no", "code", "op_id"):
            assert np.array_equal(snap.exc[f], ora.exceptions[f]), f"{what}: exception field {f}"
        assert any(v is not None for v in snap.valid), what
        run.res.free()
    report("Option", runs)
    assert_both_lanes("Option", runs)
    st.close()
    for b, _ in jobs:
        b.free()


# ---- (d) aggregates ----------------------------------------------------------------------------------------------------------
def k3_program():
    """Not a closed form (a division that can raise): the interpreting K3 kernel, with exception records."""
    sc = frontend.StageCompiler(workloads.Q6_TYPES, workloads.Q6_COLS)
    sc.add_filter(lambda x: x['l_quantity'] < 40, 100001)
    prog = sc.finish_aggregate(lambda a, x: (a[0] + x['l_quantity'] * 1000 // (x['l_shipdate'] % 13 - 6), a[1] + x['l_extended_price'] * x['l_discount']),
                               lambda a, b: (a[0] + b[0], a[1] + b[1]), (0, 0.0), 100002)
    assert prog.fused is None
    return prog


@pytest.mark.parametrize("kind", ["Q6 K3f", "K3"])
def test_aggregate_blocks_on_both_lanes(gpu, kind, monkeypatch):
    """(d) Aggregate stages, three blocks in flight: every block's partial equals the block alone and the oracle's reduction tree
    bit for bit, and K3's exception records are the oracle's."""
    monkeypatch.setenv("TPLX_JIT", "0")
    prog = workloads.q6_program() if kind == "Q6 K3f" else k3_program()
    if kind == "Q6 K3f":
        assert prog.fused is not None
    jobs, refs = [], []
    for j, n in enumerate((2_000_000, 1_500_003, 3_000_017, 999_999, 2_500_000, 1_234_567)):
        cols = workloads.gen_lineitem(n, seed=900 + j)
        blk = backend.Block.upload(0, cols, n)
        jobs.append((blk, 5 * j))
        refs.append((pyoracle.run_program(prog, cols, n, 5 * j), alone(prog, blk, 5 * j, aggregate=True)))
    st = backend.Stage(prog)
    runs = run_concurrently(st, jobs)
    for j, (run, (ora, ref)) in enumerate(zip(runs, refs)):
        what = f"{kind} block {j} (lane {run.lane})"
        snap = snapshot(run.res, aggregate=True)
        assert_same(snap, ref, what)
        assert snap.agg == ora.acc_tree, f"{what}: aggregate differs from the oracle's reduction tree"
        for f in ("row", "row_no", "code", "op_id"):
            assert np.array_equal(snap.exc[f], ora.exceptions[f]), f"{what}: exception field {f}"
        if kind == "K3":
            assert len(ora.exceptions) > 0, what
        run.res.free()
    report(kind, runs)
    assert_both_lanes(kind, runs)
    st.close()
    for b, _ in jobs:
        b.free()


# ---- (e) hash stage from several threads -------------------------------------------------------------------------------------
def keyed(n, n_keys, seed):
    rng = np.random.default_rng(seed)
    ids = rng.integers(0, n_keys, n).astype(np.int64)
    digits = np.zeros((n, 8), dtype=np.uint8)
    digits[:, 0] = ord("k")
    x = ids.copy()
    for p in range(7, 0, -1):
        digits[:, p] = ord("0") + (x % 10)
        x //= 10
    offs = (np.arange(n + 1, dtype=np.int64) * 8).astype(np.uint32)
    vi = rng.integers(-1000, 1000, n, dtype=np.int64)
    vf = rng.integers(-100000, 100000, n).astype(np.float64) / 64.0 + 0.1
    return ids, [Column(T_STR, digits.reshape(-1), offs), Column(T_I64, vi), Column(T_F64, vf)]


def ids_of(col):
    d = col.data.reshape(-1, 8)
    ids = np.zeros(len(d), dtype=np.int64)
    for p in range(1, 8):
        ids = ids * 10 + (d[:, p].astype(np.int64) - ord("0"))
    return ids


def test_hash_stage_from_several_threads_stays_on_the_primary_lane(gpu, monkeypatch):
    """(e) aggregateByKey blocks from three threads into one table: every call reports the primary lane; groups and i64 sums equal
    numpy exactly, f64 sums within n_k * eps * sum|x| (atomics: the order is not fixed)."""
    monkeypatch.setenv("TPLX_JIT", "0")
    n_keys = 200_000
    sc = frontend.StageCompiler([T_STR, T_I64, T_F64], ["key", "v", "f"])
    prog = sc.finish_hash(["key"], lambda a, x: (a[0] + x[1], a[1] + x[2]), lambda a, b: (a[0] + b[0], a[1] + b[1]), (0, 0.0), 100001)
    st = backend.Stage(prog)
    st.hash_reserve(0, n_keys)
    data = [keyed(n, n_keys, 40 + j) for j, n in enumerate((1_000_000, 700_001, 1_300_000, 500_000, 900_000, 800_017))]
    jobs = [(backend.Block.upload(0, cols, len(ids)), 0) for ids, cols in data]
    runs = run_concurrently(st, jobs)
    for r in runs:
        r.res.free()
    fin = st.hash_finish(0)
    ids = np.concatenate([d[0] for d in data])
    vi = np.concatenate([d[1][1].data for d in data])
    vf = np.concatenate([d[1][2].data for d in data])
    got = ids_of(fin.column(0))
    present = np.unique(ids)
    assert len(got) == len(present) and np.array_equal(np.sort(got), present)
    want_i = np.zeros(n_keys, dtype=np.int64)
    np.add.at(want_i, ids, vi)
    assert np.array_equal(fin.column(1).data.view(np.int64), want_i[got])
    want_f = np.bincount(ids, weights=vf, minlength=n_keys)
    abs_f = np.bincount(ids, weights=np.abs(vf), minlength=n_keys)
    cnt = np.bincount(ids, minlength=n_keys)
    bound = cnt[got] * np.finfo(np.float64).eps * abs_f[got] + 1e-300
    assert (np.abs(fin.column(2).data - want_f[got]) <= bound).all()
    assert int(fin.info.lane) == 0
    fin.free()
    report("hash", runs)
    assert {r.lane for r in runs} == {0}, "hash stages keep to the primary lane (one table per device)"
    st.close()
    for b, _ in jobs:
        b.free()


# ---- (f) run_host as bench.py step_e2e runs it -------------------------------------------------------------------------------
def test_run_host_page_locked_and_pageable_on_both_lanes(scan_case, monkeypatch):
    """(f) The prefiltered stage of (b) through tplx_gpu_stage_run_host from three threads, page-locked and pageable inputs
    alternating: page-locked late columns are read in place (zero-copy), and the non-selective block switches the prefilter off
    between other calls' upload decision and their launch."""
    prog, blocks = scan_case
    monkeypatch.setenv("TPLX_JIT", "0")
    monkeypatch.delenv("TPLX_NO_SCAN", raising=False)
    keep = []
    names = [n for n, _ in SCAN_ROUND1 + SCAN_ROUND2]
    jobs = []
    for i, name in enumerate(names):
        b = blocks[name]
        cols = pinned_columns(b["cols"], keep) if i % 2 == 0 else [Column(c.type, c.data.copy(), None if c.offsets is None else c.offsets.copy()) for c in b["cols"]]
        jobs.append((cols, b["n"], b["first"]))
    st = backend.Stage(prog)
    runs = run_host_concurrently(st, jobs)
    for i, (name, run) in enumerate(zip(names, runs)):
        b = blocks[name]
        what = f"run_host block {name} ({'page-locked' if i % 2 == 0 else 'pageable'}, lane {run.lane}, zero-copy {run.zero_copy})"
        assert_result_equals_oracle(run.res, b["ora"], what)
        assert_same(snapshot(run.res), b["ref"], what)
        if i % 2:
            assert run.zero_copy == 0, what
        run.res.free()
    zc = [names[i] for i, r in enumerate(runs) if r.zero_copy > 0]
    report("run_host", runs, extra=f"; zero-copy in {zc}")
    assert zc, "page-locked late columns must be read in place while the prefilter is on"
    assert_both_lanes("run_host", runs)
    st.close()
