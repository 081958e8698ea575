"""K9's gather (tplx_gpu_result_merge_resolved, the gather by row selector of csrc/gather.cuh) at its edges: the raw columns of a merged
result against the same rows picked on the host by `dataset._merge_by_rowno`, the restatement of ResolveTask::executeInOrder.

Sources: a stage result (A) and a block of resolved rows (B). Compared bit for bit: f64 values (NaN payloads, -0.0), bools, string
bytes and offsets (empty strings, 1 MiB strings), validity words of columns with a bitmap on neither side, only the stage side, only
the resolved side, or both; output sizes around a warp and around 2^21 rows; no normal rows, no resolved rows, every exception
resolved. The merged result's kernel launches are 1 (selectors) + 5 per string column / 1 per fixed-width column + 1 per bitmap."""
import struct

import numpy as np
import pytest

from tuplex_b200 import backend, frontend
from tuplex_b200.backend import Column, pack_valid, unpack_valid
from tuplex_b200.dataset import _merge_by_rowno
from tuplex_b200.ir import T_BOOL, T_F64, T_I64, T_STR

pytestmark = pytest.mark.gpu

IN_NAMES = ["k", "f", "b", "s", "o1", "o2", "os", "q"]
IN_TYPES = [T_I64, T_F64, T_BOOL, T_STR, T_I64, T_I64, T_STR, T_I64]
OPTION_IN = [4, 5, 6]
OUT_TYPES = [T_F64, T_BOOL, T_STR, T_I64, T_I64, T_STR, T_I64, T_I64]
# which output columns the resolved block gives a bitmap: with the stage's Option outputs 3 (o1), 4 (o2) and 5 (os) this makes
# neither side (0, 1, 6), the stage side only (3), the resolved side only (2, 7) and both sides (4, 5)
B_VALID = {2, 4, 5, 7}
FIRST_ROW_NO = 1000

F64_EDGES = [struct.unpack("<d", struct.pack("<Q", b))[0] for b in
             (0x7FF8000000000123, 0xFFF0000000000001, 0x7FF4000000000000, 0x8000000000000000, 0x7FF0000000000000, 0x0000000000000001)]


def _program():
    sc = frontend.StageCompiler(IN_TYPES, IN_NAMES, OPTION_IN)
    sc.add_map(lambda x: (x["f"], x["b"], x["s"], x["o1"], x["o2"], x["os"], x["q"] + 100 // x["k"], x["q"]), 100001)  # k == 0 raises
    return sc.finish_memory()


def _f64(rng, n):
    v = rng.standard_normal(n)
    edge = rng.random(n) < 0.2
    v[edge] = np.array(F64_EDGES)[rng.integers(0, len(F64_EDGES), int(edge.sum()))]
    return v


def _strs(rng, n, big):
    """Short strings with empty ones among them; `big`: a few 1 MiB strings as well."""
    lens = rng.integers(0, 12, n)
    lens[rng.random(n) < 0.2] = 0
    if big and n:
        lens[rng.choice(n, min(3, n), replace=False)] = 1 << 20
    offsets = np.zeros(n + 1, np.uint32)
    np.cumsum(lens, out=offsets[1:])
    return Column(T_STR, rng.integers(0, 256, int(offsets[-1])).astype(np.uint8), offsets)


def _with_valid(col, rng):
    n = len(col)
    return Column(col.type, col.data, col.offsets, pack_valid(rng.random(n) >= 0.3))


def _inputs(rng, n, exc_rows, big):
    k = rng.integers(1, 50, n).astype(np.int64)
    k[exc_rows] = 0
    return [Column(T_I64, k), Column(T_F64, _f64(rng, n)), Column(T_BOOL, rng.integers(0, 2, n).astype(np.int64)), _strs(rng, n, big),
            _with_valid(Column(T_I64, rng.integers(-1 << 62, 1 << 62, n)), rng),
            _with_valid(Column(T_I64, rng.integers(-1 << 62, 1 << 62, n)), rng), _with_valid(_strs(rng, n, big), rng),
            Column(T_I64, rng.integers(-1 << 40, 1 << 40, n))]


def _resolved(rng, n, big):
    cols = [Column(T_F64, _f64(rng, n)), Column(T_BOOL, rng.integers(0, 2, n).astype(np.int64)), _strs(rng, n, big),
            Column(T_I64, rng.integers(-1 << 62, 1 << 62, n)), Column(T_I64, rng.integers(-1 << 62, 1 << 62, n)), _strs(rng, n, big),
            Column(T_I64, rng.integers(-1 << 62, 1 << 62, n)), Column(T_I64, rng.integers(-1 << 62, 1 << 62, n))]
    return [_with_valid(c, rng) if i in B_VALID else c for i, c in enumerate(cols)]


def _pick(sel, xa, xb):
    """Per output row: xa[j] for a selector j >= 0, xb[m] for a selector ~m."""
    from_a = sel >= 0
    out = np.zeros(len(sel), np.result_type(xa, xb))
    out[from_a] = xa[sel[from_a]]
    out[~from_a] = xb[~sel[~from_a]]
    return out


def _expect_str(sel, a, b):
    """String column picked by `sel` from a and b: offsets and bytes."""
    oa, ob = a.offsets.astype(np.int64), b.offsets.astype(np.int64)
    lens = _pick(sel, oa[1:] - oa[:-1], ob[1:] - ob[:-1])
    starts = _pick(sel, oa[:-1], ob[:-1] + len(a.data))
    offsets = np.zeros(len(sel) + 1, np.int64)
    np.cumsum(lens, out=offsets[1:])
    idx = np.repeat(starts - offsets[:-1], lens) + np.arange(int(offsets[-1]))
    return offsets.astype(np.uint32), np.concatenate([a.data, b.data])[idx]


# (output rows, exception rows, resolved rows, 1 MiB strings)
CASES = [
    (31, 5, 3, False), (32, 5, 3, False), (33, 5, 3, False),
    ((1 << 21) - 1, 20000, 15000, False), ((1 << 21) + 1, 20000, 15000, False),
    (100, 10, 10, False),   # every exception resolved
    (100, 10, 0, False),    # none resolved
    (100, 0, 0, False),     # no exceptions at all
    (7, 12, 7, False),      # no normal rows
    (0, 12, 0, False),      # no normal rows and none resolved: an empty result
    (40, 8, 5, True),       # 1 MiB strings on both sides
]


@pytest.mark.parametrize("n_out,n_exc,n_res,big", CASES, ids=["out%d-exc%d-res%d%s" % (c[0], c[1], c[2], "-big" if c[3] else "") for c in CASES])
def test_merge_gather_equals_host_merge(gpu, monkeypatch, n_out, n_exc, n_res, big):
    monkeypatch.setenv("TPLX_JIT", "0")
    rng = np.random.default_rng(n_out * 7919 + n_exc * 31 + n_res)
    n = n_out + n_exc - n_res
    exc_rows = np.sort(rng.choice(n, n_exc, replace=False)) if n_exc else np.zeros(0, np.int64)
    prog = _program()
    st = backend.Stage(prog)
    blk = backend.Block.upload(0, _inputs(rng, n, exc_rows, big), n)
    res = st.run(blk, FIRST_ROW_NO)
    exc = np.sort(res.exceptions(), order="row_no")
    assert len(exc) == n_exc and int(res.info.n_out_rows) == n - n_exc
    res_nos = np.sort(rng.choice(exc["row_no"], n_res, replace=False)) if n_res else np.zeros(0, np.int64)
    rcols = _resolved(rng, n_res, big)
    rblk = backend.Block.upload(0, rcols, n_res)
    merged = res.merge_resolved(rblk, res_nos.tolist(), FIRST_ROW_NO)
    assert int(merged.info.n_out_rows) == n_out

    exc_local = exc.copy()
    exc_local["row_no"] -= FIRST_ROW_NO
    sel = np.array(_merge_by_rowno(list(range(n - n_exc)), exc_local, [(0, int(no) - FIRST_ROW_NO, ~m) for m, no in enumerate(res_nos.tolist())]),
                   np.int64)
    assert len(sel) == n_out
    launches, bitmaps = 1, set()
    for c, t in enumerate(OUT_TYPES):
        a, b, got = res.column(c), rcols[c], merged.column(c)
        b_valid = rblk.validity(c)
        bitmaps.add((a.valid is not None, b_valid is not None))
        if t == T_STR:
            want_off, want_bytes = _expect_str(sel, a, b)
            assert np.array_equal(got.offsets, want_off), f"column {c}: string offsets"
            assert np.array_equal(got.data, want_bytes), f"column {c}: string bytes"
            launches += 5
        else:
            want = _pick(sel, a.data.view(np.uint64), np.ascontiguousarray(b.data).view(np.uint64))
            assert np.array_equal(got.data.view(np.uint64), want), f"column {c}: value bits"
            launches += 1
        if a.valid is None and b_valid is None:
            assert got.valid is None, f"column {c}: a bitmap where neither source has one"
            continue
        assert got.valid is not None, f"column {c}: no bitmap"
        pa = unpack_valid(a.valid, len(a)) if a.valid is not None else np.ones(len(a), bool)
        pb = unpack_valid(b_valid, n_res) if b_valid is not None else np.ones(n_res, bool)
        present = _pick(sel, pa, pb)
        assert np.array_equal(got.valid, pack_valid(present)), f"column {c}: validity words"
        launches += 1
    assert int(merged.info.kernel_launches) == launches
    if n_res:
        assert bitmaps == {(False, False), (True, False), (False, True), (True, True)}
    merged.free()
    rblk.free()
    res.free()
    blk.free()
    st.close()
