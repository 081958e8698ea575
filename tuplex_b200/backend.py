"""ctypes binding of libtplx_gpu.so (include/tplx_gpu.h) + host column blocks.

This is the host-side mirror of the reference's backend plug-in point
(IBackend::execute, tuplex/core/include/ee/IBackend.h:29-46; selected by `tuplex.backend`,
tuplex/core/src/Context.cc:56-83). There is deliberately no CPU implementation behind it: if the CUDA
library is missing or no device is visible every call raises GpuBackendError.
"""
from __future__ import annotations

import ctypes as ct
import os
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from . import ir
from .ir import T_BOOL, T_F64, T_I64, T_STR

_LIB_PATH = os.environ.get("TPLX_GPU_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libtplx_gpu.so")
MAX_COLS = ir.C["TPLX_MAX_COLS"]
E_NOMEM = -5  # TPLX_E_NOMEM
CONCAT_DROP_VALID, CONCAT_ALL_NONE, CONCAT_UTF8 = 1, 2, 4  # tplx_concat_flags


class GpuBackendError(RuntimeError):
    code = 0  # tplx_status of the failed call (0 = not from the C ABI)


class CColumn(ct.Structure):
    _fields_ = [("type", ct.c_uint8), ("pad", ct.c_uint8 * 7), ("data", ct.c_void_p), ("offsets", ct.c_void_p),
                ("data_bytes", ct.c_uint64), ("valid", ct.c_void_p)]


class CExceptionRec(ct.Structure):
    _fields_ = [("row", ct.c_int64), ("row_no", ct.c_int64), ("code", ct.c_int64), ("op_id", ct.c_int64)]


class CResultInfo(ct.Structure):
    _fields_ = [("n_in_rows", ct.c_uint64), ("n_out_rows", ct.c_uint64), ("n_exceptions", ct.c_uint64),
                ("out_str_bytes", ct.c_uint64 * MAX_COLS), ("kernel_ms", ct.c_double), ("total_ms", ct.c_double),
                ("kernel_launches", ct.c_uint32), ("zero_copy_cols", ct.c_uint32), ("h2d_bytes", ct.c_uint64),
                ("specialised_launches", ct.c_uint32), ("lane", ct.c_uint32)]


class CCsvDesc(ct.Structure):
    _fields_ = [("delimiter", ct.c_uint8), ("quotechar", ct.c_uint8), ("skip_header", ct.c_uint8), ("n_null_values", ct.c_uint8),
                ("n_file_cols", ct.c_uint32), ("col_types", ct.c_char_p), ("null_values", ct.POINTER(ct.c_char_p)),
                ("col_lazy", ct.c_char_p)]


class CCsvInfo(ct.Structure):
    _fields_ = [("n_rows", ct.c_uint64), ("n_normal", ct.c_uint64), ("n_bad", ct.c_uint64), ("sequential_rows", ct.c_uint32),
                ("kernel_launches", ct.c_uint32), ("parse_ms", ct.c_double)]


class CConcatPiece(ct.Structure):
    _fields_ = [("block", ct.c_void_p), ("first_row", ct.c_uint64), ("n_rows", ct.c_uint64)]


class CTextDesc(ct.Structure):
    _fields_ = [("n_null_values", ct.c_uint8), ("option", ct.c_uint8), ("null_values", ct.POINTER(ct.c_char_p))]


CSV_SKIP = 0xFF
CSV_BAD_DTYPE = np.dtype([("row", "<u4"), ("code", "<u4"), ("line_start", "<u4"), ("line_end", "<u4")])
EXC_DTYPE = np.dtype([("row", "<i8"), ("row_no", "<i8"), ("code", "<i8"), ("op_id", "<i8")])

_lib = None


def lib():
    """Load the CUDA library; fails loudly (no fallback) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise GpuBackendError(f"{_LIB_PATH} not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                              "the GPU backend has no CPU fallback")
    L = ct.CDLL(_LIB_PATH)
    vp, i32, u32, u64, i64 = ct.c_void_p, ct.c_int32, ct.c_uint32, ct.c_uint64, ct.c_int64
    P = ct.POINTER
    sig = {
        "tplx_gpu_init": ([P(i32), i32], i32),
        "tplx_gpu_device_count": ([], i32),
        "tplx_gpu_shutdown": ([], i32),
        "tplx_gpu_last_error": ([], ct.c_char_p),
        "tplx_gpu_device_info": ([i32, ct.c_char_p, i32, P(i32), P(u64)], i32),
        "tplx_gpu_stage_create": ([vp, u64, P(vp)], i32),
        "tplx_gpu_stage_destroy": ([vp], i32),
        "tplx_gpu_stage_vec_plan": ([vp, vp, u32, P(u32), P(u32), vp, u32], i32),
        "tplx_gpu_stage_specialise": ([vp, i32, i32, ct.c_char_p, u64, P(u64), P(u64), ct.c_char_p, u64], i32),
        "tplx_gpu_block_upload": ([i32, P(CColumn), u32, u64, P(vp)], i32),
        "tplx_gpu_block_wrap_device": ([i32, P(CColumn), u32, u64, P(vp)], i32),
        "tplx_gpu_block_from_partitions": ([i32, P(vp), P(u64), u32, P(ct.c_uint8), u32, P(vp)], i32),
        "tplx_gpu_block_rows": ([vp, P(u64)], i32),
        "tplx_gpu_block_column_bytes": ([vp, P(u64), u32, P(u32)], i32),
        "tplx_gpu_block_fetch_validity": ([vp, u32, vp, P(u32)], i32),
        "tplx_gpu_block_free": ([vp], i32),
        "tplx_gpu_block_concat": ([P(vp), u32, P(vp)], i32),
        "tplx_gpu_block_concat_pieces": ([P(CConcatPiece), u32, vp, P(vp)], i32),
        "tplx_gpu_block_stats": ([vp, P(u64), P(u64)], i32),
        "tplx_gpu_block_fetch_column": ([vp, u32, vp, vp], i32),
        "tplx_gpu_block_view": ([vp, P(vp)], i32),
        "tplx_gpu_block_select": ([vp, vp, P(vp)], i32),
        "tplx_gpu_block_device_column": ([vp, u32, P(vp), P(vp), P(vp), P(u64)], i32),
        "tplx_gpu_stage_run": ([vp, vp, i64, P(vp)], i32),
        "tplx_gpu_stage_run_host": ([vp, i32, P(CColumn), u32, u64, i64, P(vp)], i32),
        "tplx_gpu_result_info": ([vp, P(CResultInfo)], i32),
        "tplx_gpu_result_fetch_column": ([vp, u32, vp, vp], i32),
        "tplx_gpu_result_device_column": ([vp, u32, P(vp), P(vp)], i32),
        "tplx_gpu_result_fetch_exceptions": ([vp, vp], i32),
        "tplx_gpu_result_fetch_aggregate": ([vp, P(i64)], i32),
        "tplx_gpu_result_partitions": ([vp, u64, vp, u64, P(u64), P(u64), u32, P(u32)], i32),
        "tplx_gpu_result_exception_partition": ([vp, vp, u64, P(u64)], i32),
        "tplx_gpu_result_csv": ([vp, u32, ct.c_uint8, ct.c_uint8, vp, u64, P(u64)], i32),
        "tplx_gpu_result_csv_nulls": ([vp, u32, ct.c_uint8, ct.c_uint8, ct.c_char_p, vp, u64, P(u64)], i32),
        "tplx_gpu_result_free": ([vp], i32),
        "tplx_gpu_stage_hash_reserve": ([vp, i32, u64], i32),
        "tplx_gpu_stage_hash_finish": ([vp, i32, P(vp)], i32),
        "tplx_gpu_stage_hash_export_raw": ([vp, i32, P(vp)], i32),
        "tplx_gpu_stage_hash_merge": ([vp, vp], i32),
        "tplx_gpu_stage_hash_reset": ([vp, i32], i32),
        "tplx_gpu_join_build": ([vp, u32, P(vp)], i32),
        "tplx_gpu_join_info": ([vp, P(u64), P(u64), P(ct.c_double), P(u32)], i32),
        "tplx_gpu_join_probe": ([vp, vp, u32, u32, P(vp)], i32),
        "tplx_gpu_join_destroy": ([vp], i32),
        "tplx_gpu_result_fetch_validity": ([vp, u32, vp, P(u32)], i32),
        "tplx_gpu_result_device_validity": ([vp, u32, P(vp)], i32),
        "tplx_gpu_result_merge_resolved": ([vp, vp, P(i64), i64, P(vp)], i32),
        "tplx_gpu_result_sort_by_keys": ([vp, u32, ct.c_char_p, P(vp)], i32),
        "tplx_gpu_comm_unique_id": ([vp], i32),
        "tplx_gpu_comm_init": ([i32, i32, i32, vp], i32),
        "tplx_gpu_comm_init_local": ([P(i32), i32], i32),
        "tplx_gpu_comm_info": ([i32, P(i32), P(i32)], i32),
        "tplx_gpu_comm_destroy": ([i32], i32),
        "tplx_gpu_agg_finish": ([vp, i32, P(i64), P(i64)], i32),
        "tplx_gpu_stage_hash_exchange": ([vp, i32], i32),
        "tplx_gpu_csv_upload": ([i32, vp, u64, P(vp)], i32),
        "tplx_gpu_csv_buffer_free": ([vp], i32),
        "tplx_gpu_csv_parse": ([vp, P(CCsvDesc), P(vp), P(vp)], i32),
        "tplx_gpu_csv_result_info": ([vp, P(CCsvInfo)], i32),
        "tplx_gpu_csv_result_fetch_bad_rows": ([vp, vp], i32),
        "tplx_gpu_csv_result_fetch_rowmap": ([vp, vp], i32),
        "tplx_gpu_csv_result_fetch_row_ends": ([vp, vp], i32),
        "tplx_gpu_csv_result_free": ([vp], i32),
        "tplx_gpu_text_parse": ([vp, P(CTextDesc), P(vp), P(vp)], i32),
    }
    for name, (argtypes, restype) in sig.items():
        fn = getattr(L, name)  # AttributeError if the library does not export a declared symbol
        fn.argtypes = argtypes
        fn.restype = restype
    L._declared = sorted(sig)
    _lib = L
    return L


def _check(rc: int, what: str):
    if rc != 0:
        msg = lib().tplx_gpu_last_error().decode("utf-8", "replace")
        err = GpuBackendError(f"{what} failed ({rc}): {msg}")
        err.code = rc
        raise err


_initialised: set = set()


def init(devices: Optional[Sequence[int]] = None):
    L = lib()
    devs = list(devices) if devices else [0]
    if set(devs) <= _initialised:
        return
    arr = (ct.c_int32 * len(devs))(*devs)
    _check(L.tplx_gpu_init(arr, len(devs)), "tplx_gpu_init")
    _initialised.update(devs)


def device_count() -> int:
    return lib().tplx_gpu_device_count()


# ---- communicator (the one exchange step of the path; include/tplx_gpu.h "multi-GPU") -------------------------------
COMM_ID_BYTES = ir.C["TPLX_COMM_ID_BYTES"]


def comm_unique_id() -> bytes:
    buf = ct.create_string_buffer(COMM_ID_BYTES)
    _check(lib().tplx_gpu_comm_unique_id(buf), "tplx_gpu_comm_unique_id")
    return buf.raw


def comm_init(device: int, rank: int, world: int, uid: bytes):
    """Collective over all ranks (one rank per process and device)."""
    init([device])
    buf = ct.create_string_buffer(bytes(uid), COMM_ID_BYTES)
    _check(lib().tplx_gpu_comm_init(device, rank, world, buf), "tplx_gpu_comm_init")


def comm_init_local(devices: Sequence[int]):
    """One process driving several devices: rank = position in `devices`."""
    init(devices)
    arr = (ct.c_int32 * len(devices))(*devices)
    _check(lib().tplx_gpu_comm_init_local(arr, len(devices)), "tplx_gpu_comm_init_local")


def comm_info(device: int):
    r, w = ct.c_int32(), ct.c_int32()
    rc = lib().tplx_gpu_comm_info(device, ct.byref(r), ct.byref(w))
    return (r.value, w.value) if rc == 0 else None


def comm_destroy(device: int):
    lib().tplx_gpu_comm_destroy(device)


# ------------------------------------------------------------------------------------------------
# host column blocks
# ------------------------------------------------------------------------------------------------
def pack_valid(present: np.ndarray) -> np.ndarray:
    """bool per row -> validity words (bit (r & 31) of word r >> 5)."""
    n = len(present)
    bits = np.zeros(((n + 31) // 32) * 32, dtype=np.uint8)
    bits[:n] = present
    return np.packbits(bits.reshape(-1, 32), axis=1, bitorder="little").view("<u4").reshape(-1).copy()


def unpack_valid(words: np.ndarray, n: int) -> np.ndarray:
    return np.unpackbits(np.ascontiguousarray(words, dtype="<u4").view(np.uint8), bitorder="little")[:n].astype(bool)


@dataclass
class Column:
    """One column of a column block on the host. Fixed width: `data` is an 8-byte numpy array
    (int64 / float64; bool stored as int64 0/1). Strings: `data` = uint8 bytes, `offsets` = uint32[n+1]."""
    type: int
    data: np.ndarray
    offsets: Optional[np.ndarray] = None
    valid: Optional[np.ndarray] = None  # Option[T] column: uint32 words, bit (r & 31) of word r >> 5 set = row r holds a value; None = no Nones

    def __len__(self):
        return len(self.offsets) - 1 if self.type == T_STR else len(self.data)

    @staticmethod
    def from_values(values: Sequence, t: int) -> "Column":
        """Values of one type; None entries make the column an Option[T] column (validity bitmap, placeholder value 0 / '')."""
        valid = None
        if any(v is None for v in values):
            present = np.fromiter((v is not None for v in values), dtype=bool, count=len(values))
            valid = pack_valid(present)
            fill = "" if t == T_STR else 0
            values = [fill if v is None else v for v in values]
        if t == T_STR:
            enc = [v.encode("utf-8") for v in values]
            lens = np.fromiter((len(b) for b in enc), dtype=np.int64, count=len(enc))
            offsets = np.zeros(len(enc) + 1, dtype=np.uint32)
            np.cumsum(lens, out=offsets[1:])
            if lens.sum() > 0xFFFFFFFF:
                raise GpuBackendError("string column exceeds 4 GiB; use smaller blocks")
            data = np.frombuffer(b"".join(enc), dtype=np.uint8).copy() if enc else np.zeros(0, np.uint8)
            return Column(T_STR, data, offsets, valid)
        if t == T_F64:
            return Column(T_F64, np.asarray(values, dtype=np.float64), None, valid)
        return Column(t, np.asarray(values, dtype=np.int64), None, valid)

    def present(self) -> Optional[np.ndarray]:
        """bool per row (True = holds a value), or None for a column without Nones."""
        return None if self.valid is None else unpack_valid(self.valid, len(self))

    def to_values(self) -> list:
        if self.type == T_STR:
            raw = self.data.tobytes()
            o = self.offsets
            # device string ops are byte based (ASCII case mapping, byte slices): a slice may cut a multi-byte sequence. Decode like
            # csvsource._text does, so that such a cell becomes a row value instead of failing the whole collect()
            vals = [raw[o[i]:o[i + 1]].decode("utf-8", "replace") for i in range(len(o) - 1)]
        elif self.type == T_BOOL:
            vals = [bool(v) for v in self.data.tolist()]
        else:
            vals = self.data.tolist()
        if self.valid is not None:
            vals = [v if ok else None for v, ok in zip(vals, self.present().tolist())]
        return vals

    def slice(self, lo: int, hi: int) -> "Column":
        valid = None if self.valid is None else pack_valid(self.present()[lo:hi])
        if self.type == T_STR:
            o = self.offsets[lo:hi + 1]
            return Column(T_STR, self.data[int(o[0]):int(o[-1])], (o - o[0]).astype(np.uint32), valid)
        return Column(self.type, self.data[lo:hi], None, valid)

    def take(self, idx: np.ndarray) -> "Column":
        if self.type == T_STR:
            vals = self.to_values()
            return Column.from_values([vals[i] for i in idx.tolist()], T_STR)
        valid = None if self.valid is None else pack_valid(self.present()[idx])
        return Column(self.type, self.data[idx], None, valid)

    def nbytes(self) -> int:
        return int(self.data.nbytes + (self.offsets.nbytes if self.offsets is not None else 0))


def _ccols(cols: Sequence[Column]):
    arr = (CColumn * max(len(cols), 1))()
    keep = []
    for i, c in enumerate(cols):
        d = np.ascontiguousarray(c.data)
        keep.append(d)
        arr[i].type = c.type
        arr[i].data = d.ctypes.data
        if c.type == T_STR:
            o = np.ascontiguousarray(c.offsets, dtype=np.uint32)
            keep.append(o)
            arr[i].offsets = o.ctypes.data
            arr[i].data_bytes = int(o[-1]) if len(o) else 0
        else:
            arr[i].offsets = None
            arr[i].data_bytes = d.nbytes
        if c.valid is not None:
            v = np.ascontiguousarray(c.valid, dtype=np.uint32)
            keep.append(v)
            arr[i].valid = v.ctypes.data
        else:
            arr[i].valid = None
    return arr, keep


class Stage:
    """Device-side stage handle (replaces TransformStage + its JIT-compiled functor)."""

    def __init__(self, program: ir.Program):
        self.program = program
        blob = program.serialize()
        self._h = ct.c_void_p()
        buf = ct.create_string_buffer(blob, len(blob))
        _check(lib().tplx_gpu_stage_create(buf, len(blob), ct.byref(self._h)), "tplx_gpu_stage_create")

    def vec_plan(self):
        """(micro-ops, n_slots, output slots) of the fixed-width row kernel for this stage, or None when it is not eligible
        (tplx_gpu_stage_vec_plan; no device needed). Micro-ops are dicts with the fields of tplx_vec_uop."""
        n, ns = ct.c_uint32(), ct.c_uint32()
        _check(lib().tplx_gpu_stage_vec_plan(self._h, None, 0, ct.byref(n), ct.byref(ns), None, 0), "tplx_gpu_stage_vec_plan")
        if n.value == 0:
            return None
        dt = np.dtype([("vop", "<u4"), ("xflags", "<u4"), ("flags", "u1"), ("pad0", "u1"), ("opidx", "<u2"), ("dst", "<u2"), ("a", "<u2"),
                       ("b", "<u2"), ("c", "<u2"), ("guard", "<u2"), ("pad1", "<u2"), ("imm", "<i8"), ("imm2", "<i8")])
        assert dt.itemsize == 40
        buf = np.zeros(n.value, dt)
        n_out = len(self.program.out_cols)
        outs = np.zeros(max(n_out, 1), np.uint16)
        _check(lib().tplx_gpu_stage_vec_plan(self._h, buf.ctypes.data, n.value, ct.byref(n), ct.byref(ns), outs.ctypes.data, n_out),
               "tplx_gpu_stage_vec_plan")
        uops = [{k: int(r[k]) for k in dt.names if not k.startswith("pad")} for r in buf]
        return uops, ns.value, [int(x) for x in outs[:n_out]]

    def specialise(self, kind: int, compile: bool = True):
        """(generated CUDA row function, cubin size, compiler log) of the stage specialiser for kernel `kind`
        (tplx_gpu_stage_specialise; needs no device). cubin size 0 = NVRTC absent or the compile failed (see the log)."""
        n, nb = ct.c_uint64(), ct.c_uint64()
        src = ct.create_string_buffer(1 << 20)
        log = ct.create_string_buffer(1 << 16)
        _check(lib().tplx_gpu_stage_specialise(self._h, kind, 1 if compile else 0, src, len(src), ct.byref(n), ct.byref(nb), log, len(log)),
               "tplx_gpu_stage_specialise")
        return src.value.decode(), int(nb.value), log.value.decode(errors="replace")

    def close(self):
        if self._h:
            lib().tplx_gpu_stage_destroy(self._h)
            self._h = ct.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- blocks --
    def upload(self, device: int, cols: Sequence[Column], n_rows: int) -> "Block":
        return Block.upload(device, cols, n_rows)

    def run(self, block: "Block", first_row_no: int = 0) -> "Result":
        h = ct.c_void_p()
        _check(lib().tplx_gpu_stage_run(self._h, block._h, first_row_no, ct.byref(h)), "tplx_gpu_stage_run")
        return Result(h, self, block)

    def run_host(self, device: int, cols: Sequence[Column], n_rows: int, first_row_no: int = 0) -> "Result":
        arr, keep = _ccols(cols)
        h = ct.c_void_p()
        _check(lib().tplx_gpu_stage_run_host(self._h, device, arr, len(cols), n_rows, first_row_no, ct.byref(h)),
               "tplx_gpu_stage_run_host")
        r = Result(h, self, None)
        r._keep = keep
        r.device = device
        return r

    def agg_finish(self, device: int, local_bits: Sequence[int]) -> List[int]:
        """Collective: combine this rank's partial aggregate with every other rank's, in rank order (tplx_gpu_agg_finish)."""
        n = len(self.program.accs)
        src = (ct.c_int64 * n)(*[ir._as_i64(b) for b in local_bits])
        dst = (ct.c_int64 * n)()
        _check(lib().tplx_gpu_agg_finish(self._h, device, src, dst), "tplx_gpu_agg_finish")
        return [v & ((1 << 64) - 1) for v in dst]

    def hash_exchange(self, device: int):
        """Collective: hash-partitioned all-to-all of the per-rank tables; afterwards hash_finish yields the groups this
        rank owns (tplx_gpu_stage_hash_exchange)."""
        _check(lib().tplx_gpu_stage_hash_exchange(self._h, device), "tplx_gpu_stage_hash_exchange")

    def hash_reserve(self, device: int, expected_keys: int):
        _check(lib().tplx_gpu_stage_hash_reserve(self._h, device, expected_keys), "tplx_gpu_stage_hash_reserve")

    def hash_finish(self, device: int, raw: bool = False) -> "Result":
        h = ct.c_void_p()
        fn = lib().tplx_gpu_stage_hash_export_raw if raw else lib().tplx_gpu_stage_hash_finish
        _check(fn(self._h, device, ct.byref(h)), "tplx_gpu_stage_hash_finish")
        return Result(h, self, None, hash_result=True)

    def hash_merge(self, packed: "Block"):
        _check(lib().tplx_gpu_stage_hash_merge(self._h, packed._h), "tplx_gpu_stage_hash_merge")

    def hash_reset(self, device: int):
        _check(lib().tplx_gpu_stage_hash_reset(self._h, device), "tplx_gpu_stage_hash_reset")


class Block:
    def __init__(self, h, n_rows, device, keep=None):
        self._h = h
        self.n_rows = n_rows
        self.device = device
        self._keep = keep

    @staticmethod
    def upload(device: int, cols: Sequence[Column], n_rows: int) -> "Block":
        init([device])
        arr, keep = _ccols(cols)
        h = ct.c_void_p()
        _check(lib().tplx_gpu_block_upload(device, arr, len(cols), n_rows, ct.byref(h)), "tplx_gpu_block_upload")
        return Block(h, n_rows, device, keep)

    @staticmethod
    def wrap_device(device: int, ptr_cols: Sequence[tuple], n_rows: int, keep=None) -> "Block":
        """ptr_cols: (type, data_ptr, offsets_ptr or 0, data_bytes[, valid_ptr or 0]) with device addresses; `keep` is held as long
        as the block (the owner of the memory)."""
        init([device])
        arr = (CColumn * max(len(ptr_cols), 1))()
        for i, (t, dp, op, nb, *vp) in enumerate(ptr_cols):
            arr[i].type = t
            arr[i].data = dp
            arr[i].offsets = op or None
            arr[i].data_bytes = nb
            arr[i].valid = (vp[0] if vp else 0) or None
        h = ct.c_void_p()
        _check(lib().tplx_gpu_block_wrap_device(device, arr, len(ptr_cols), n_rows, ct.byref(h)), "tplx_gpu_block_wrap_device")
        return Block(h, n_rows, device, keep)

    @staticmethod
    def concat(parts: Sequence["Block"]) -> "Block":
        """The rows of `parts` in order as one new block that owns its memory (tplx_gpu_block_concat); the parts may be freed
        afterwards."""
        if parts:
            init([parts[0].device])
        arr = (ct.c_void_p * max(len(parts), 1))(*[p._h for p in parts])
        h = ct.c_void_p()
        _check(lib().tplx_gpu_block_concat(arr, len(parts), ct.byref(h)), "tplx_gpu_block_concat")
        nr = ct.c_uint64()
        _check(lib().tplx_gpu_block_rows(h, ct.byref(nr)), "tplx_gpu_block_rows")
        return Block(h, nr.value, parts[0].device if parts else 0)

    @staticmethod
    def concat_pieces(pieces: Sequence[tuple], col_flags: Optional[Sequence[int]] = None) -> "Block":
        """Rows [first, first + n) of every (block, first, n) piece, in order, as one new block that owns its memory
        (tplx_gpu_block_concat_pieces); `col_flags` holds one CONCAT_* combination per column (None: every column as concat makes
        it). The blocks may be freed afterwards."""
        if pieces:
            init([pieces[0][0].device])
        arr = (CConcatPiece * max(len(pieces), 1))()
        for i, (b, first, n) in enumerate(pieces):
            arr[i].block, arr[i].first_row, arr[i].n_rows = b._h, int(first), int(n)
        flags = bytes(col_flags) if col_flags is not None else None
        h = ct.c_void_p()
        _check(lib().tplx_gpu_block_concat_pieces(arr, len(pieces), flags, ct.byref(h)), "tplx_gpu_block_concat_pieces")
        nr = ct.c_uint64()
        _check(lib().tplx_gpu_block_rows(h, ct.byref(nr)), "tplx_gpu_block_rows")
        return Block(h, nr.value, pieces[0][0].device if pieces else 0)

    def n_cols(self) -> int:
        n = ct.c_uint32()
        _check(lib().tplx_gpu_block_column_bytes(self._h, None, 0, ct.byref(n)), "tplx_gpu_block_column_bytes")
        return n.value

    def column_bytes(self) -> List[int]:
        """Device bytes of every column: values, or string bytes + offsets (tplx_gpu_block_column_bytes); bitmaps not included."""
        arr = (ct.c_uint64 * MAX_COLS)()
        n = ct.c_uint32()
        _check(lib().tplx_gpu_block_column_bytes(self._h, arr, MAX_COLS, ct.byref(n)), "tplx_gpu_block_column_bytes")
        return [int(arr[i]) for i in range(n.value)]

    def stats(self):
        """(None rows, strings that are not valid UTF-8) per column, counted on the device (tplx_gpu_block_stats)."""
        none, bad = (ct.c_uint64 * MAX_COLS)(), (ct.c_uint64 * MAX_COLS)()
        _check(lib().tplx_gpu_block_stats(self._h, none, bad), "tplx_gpu_block_stats")
        n = self.n_cols()
        return [int(none[i]) for i in range(n)], [int(bad[i]) for i in range(n)]

    def column(self, c: int, t: int) -> "Column":
        """Column c (of type t) fetched to the host with its validity words, tail bits cleared (tplx_gpu_block_fetch_column)."""
        n = int(self.n_rows)
        valid = self.validity(c)
        if valid is not None and n & 31:
            valid[-1] &= np.uint32((1 << (n & 31)) - 1)
        if t == T_STR:
            offsets = np.empty(n + 1, dtype=np.uint32)
            _check(lib().tplx_gpu_block_fetch_column(self._h, c, None, offsets.ctypes.data), "block_fetch_column")
            data = np.empty(max(int(offsets[-1]), 1), dtype=np.uint8)
            _check(lib().tplx_gpu_block_fetch_column(self._h, c, data.ctypes.data, None), "block_fetch_column")
            return Column(T_STR, data[:int(offsets[-1])], offsets, valid)
        data = np.empty(n, dtype=np.float64 if t == T_F64 else np.int64)
        if n:
            _check(lib().tplx_gpu_block_fetch_column(self._h, c, data.ctypes.data, None), "block_fetch_column")
        return Column(t, data, None, valid)

    def view(self) -> "Block":
        """A block over this block's memory that owns none of it (tplx_gpu_block_view): freeing it leaves this block intact."""
        h = ct.c_void_p()
        _check(lib().tplx_gpu_block_view(self._h, ct.byref(h)), "tplx_gpu_block_view")
        return Block(h, self.n_rows, self.device, keep=self)

    def select(self, keep_words: np.ndarray) -> "Block":
        """The rows whose bit is set in `keep_words` (bit r & 31 of word r >> 5), in order, as a new block that owns its memory
        (tplx_gpu_block_select); this block may be freed afterwards."""
        words = np.ascontiguousarray(keep_words, dtype=np.uint32)
        if len(words) != (int(self.n_rows) + 31) // 32:
            raise ValueError("select: one keep word per 32 rows")
        h = ct.c_void_p()
        _check(lib().tplx_gpu_block_select(self._h, words.ctypes.data if len(words) else None, ct.byref(h)), "tplx_gpu_block_select")
        nr = ct.c_uint64()
        _check(lib().tplx_gpu_block_rows(h, ct.byref(nr)), "tplx_gpu_block_rows")
        return Block(h, nr.value, self.device)

    def device_column(self, c: int, t: int) -> tuple:
        """Column c (of type t) as Block.wrap_device takes it: (type, data, offsets, data_bytes, validity), device addresses
        (tplx_gpu_block_device_column); this block must outlive their use."""
        d, o, v, nb = ct.c_void_p(), ct.c_void_p(), ct.c_void_p(), ct.c_uint64()
        _check(lib().tplx_gpu_block_device_column(self._h, c, ct.byref(d), ct.byref(o), ct.byref(v), ct.byref(nb)), "tplx_gpu_block_device_column")
        return t, d.value or 0, o.value or 0, int(nb.value), v.value or 0

    @staticmethod
    def from_partitions(device: int, partitions: Sequence[bytes], col_types: Sequence[int], option_cols: Sequence[int] = ()) -> "Block":
        """option_cols: Option[T] fields of the schema (they take part in the row bitmap, Serializer.cc:1041-1059)."""
        init([device])
        col_types = [t | (ir.C["TPLX_T_OPTION"] if c in set(option_cols) else 0) for c, t in enumerate(col_types)]
        n = len(partitions)
        bufs = [np.frombuffer(p, dtype=np.uint8) for p in partitions]
        ptrs = (ct.c_void_p * max(n, 1))(*[b.ctypes.data for b in bufs])
        sizes = (ct.c_uint64 * max(n, 1))(*[len(p) for p in partitions])
        types = (ct.c_uint8 * len(col_types))(*col_types)
        h = ct.c_void_p()
        _check(lib().tplx_gpu_block_from_partitions(device, ptrs, sizes, n, types, len(col_types), ct.byref(h)),
               "tplx_gpu_block_from_partitions")
        nr = ct.c_uint64()
        _check(lib().tplx_gpu_block_rows(h, ct.byref(nr)), "tplx_gpu_block_rows")
        return Block(h, nr.value, device)

    def validity(self, c: int) -> Optional[np.ndarray]:
        """Validity words of an Option[T] column as the block stores them, tail bits included (tplx_gpu_block_fetch_validity);
        None for a column without a bitmap."""
        nullable = ct.c_uint32()
        _check(lib().tplx_gpu_block_fetch_validity(self._h, c, None, ct.byref(nullable)), "block_fetch_validity")
        if not nullable.value:
            return None
        words = np.zeros((int(self.n_rows) + 31) // 32, dtype=np.uint32)
        if len(words):
            _check(lib().tplx_gpu_block_fetch_validity(self._h, c, words.ctypes.data, ct.byref(nullable)), "block_fetch_validity")
        return words

    def free(self):
        if self._h:
            lib().tplx_gpu_block_free(self._h)
            self._h = ct.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Result:
    def __init__(self, h, stage: Optional[Stage], block: Optional[Block], hash_result: bool = False, types: Optional[List[int]] = None):
        self._h = h
        self.stage = stage
        self.block = block  # keep the input alive for exception gather
        self._info = None
        self.hash_result = hash_result
        self._types = types  # results that do not come from a stage (join probe): the output column types
        self._rowidx: Optional[bool] = None
        self.device = block.device if block is not None else None

    @property
    def info(self) -> CResultInfo:
        if self._info is None:
            inf = CResultInfo()
            _check(lib().tplx_gpu_result_info(self._h, ct.byref(inf)), "tplx_gpu_result_info")
            self._info = inf
        return self._info

    def out_types(self) -> List[int]:
        if self._types is not None:
            return list(self._types)
        p = self.stage.program
        if self.hash_result:
            f = {ir.C["TPLX_ACC_SUM_F64"], ir.C["TPLX_ACC_MIN_F64"], ir.C["TPLX_ACC_MAX_F64"]}
            return [t for _, t in p.out_cols[: p.n_keys]] + [T_F64 if a.kind in f else T_I64 for a in p.accs]
        return [t for _, t in p.out_cols][: len(p.out_cols) - p.hidden_out_cols]

    def column(self, c: int) -> Column:
        t = self.out_types()[c]
        n = int(self.info.n_out_rows)
        if t == T_STR:
            nb = int(self.info.out_str_bytes[c])
            data = np.empty(max(nb, 1), dtype=np.uint8)
            offsets = np.empty(n + 1, dtype=np.uint32)
            _check(lib().tplx_gpu_result_fetch_column(self._h, c, data.ctypes.data, offsets.ctypes.data), "result_fetch_column")
            return Column(T_STR, data[:nb], offsets, self.validity(c))
        data = np.empty(n, dtype=np.float64 if t == T_F64 else np.int64)
        if n:
            _check(lib().tplx_gpu_result_fetch_column(self._h, c, data.ctypes.data, None), "result_fetch_column")
        return Column(t, data, None, self.validity(c))

    def validity(self, c: int) -> Optional[np.ndarray]:
        """Validity words of a nullable output column (tplx_gpu_result_fetch_validity), None for a column that cannot hold None."""
        nullable = ct.c_uint32()
        _check(lib().tplx_gpu_result_fetch_validity(self._h, c, None, ct.byref(nullable)), "result_fetch_validity")
        if not nullable.value:
            return None
        n = int(self.info.n_out_rows)
        words = np.zeros((n + 31) // 32, dtype=np.uint32)
        if n:
            _check(lib().tplx_gpu_result_fetch_validity(self._h, c, words.ctypes.data, ct.byref(nullable)), "result_fetch_validity")
            if n & 31:
                words[-1] &= np.uint32((1 << (n & 31)) - 1)
        return words

    def columns(self) -> List[Column]:
        return [self.column(c) for c in range(len(self.out_types()))]

    def as_block(self, n_cols: Optional[int] = None) -> Block:
        """The first `n_cols` visible output columns (default: all but a stage's trailing __rowidx) as a block, with their
        validity bitmaps, without a copy; the block keeps this result alive."""
        types = self.out_types()
        if n_cols is None:
            n_cols = len(types) - (1 if self.rowidx else 0)
        n = int(self.info.n_out_rows)
        cols = []
        for c in range(n_cols):
            dp, op = self.device_column(c)
            w = ct.c_void_p()
            _check(lib().tplx_gpu_result_device_validity(self._h, c, ct.byref(w)), "result_device_validity")
            cols.append((types[c], dp, op, int(self.info.out_str_bytes[c]) if types[c] == T_STR else n * 8, w.value or 0))
        return Block.wrap_device(self.device, cols, n, keep=self)

    @property
    def rowidx(self) -> bool:
        """The last visible output column is the stage's __rowidx (input row numbers), not a user column."""
        if self._rowidx is None:
            p = self.stage.program if self.stage is not None else None
            self._rowidx = bool(p is not None and not self.hash_result and p.out_names[len(self.out_types()) - 1:len(self.out_types())] == ["__rowidx"])
        return self._rowidx

    def device_column(self, c: int):
        d, o = ct.c_void_p(), ct.c_void_p()
        _check(lib().tplx_gpu_result_device_column(self._h, c, ct.byref(d), ct.byref(o)), "result_device_column")
        return d.value or 0, o.value or 0

    def exceptions(self) -> np.ndarray:
        n = int(self.info.n_exceptions)
        recs = np.zeros(n, dtype=EXC_DTYPE)
        if n:
            _check(lib().tplx_gpu_result_fetch_exceptions(self._h, recs.ctypes.data), "result_fetch_exceptions")
        return recs

    def aggregate_bits(self) -> List[int]:
        n = len(self.stage.program.accs)
        arr = (ct.c_int64 * n)()
        _check(lib().tplx_gpu_result_fetch_aggregate(self._h, arr), "result_fetch_aggregate")
        return [v & ((1 << 64) - 1) for v in arr]

    def partitions(self, partition_bytes: int = 32 << 20) -> List[bytes]:
        need, nparts = ct.c_uint64(), ct.c_uint32()
        _check(lib().tplx_gpu_result_partitions(self._h, partition_bytes, None, 0, ct.byref(need), None, 0, ct.byref(nparts)),
               "result_partitions(size)")
        buf = np.empty(max(need.value, 8), dtype=np.uint8)
        offs = (ct.c_uint64 * (nparts.value + 1))()
        _check(lib().tplx_gpu_result_partitions(self._h, partition_bytes, buf.ctypes.data, buf.nbytes, ct.byref(need), offs,
                                                nparts.value, ct.byref(nparts)), "result_partitions")
        raw = buf.tobytes()
        return [raw[offs[p]:offs[p + 1]] for p in range(nparts.value)]

    def csv_bytes(self, delimiter=",", quotechar='"', n_cols: int = 0, null_value: Optional[str] = None) -> Optional[bytes]:
        """First n_cols (0 = all) output columns as CSV text written on the device (K7); None when an f64 cell has a magnitude
        >= 2^63 (TPLX_E_UNSUPPORTED: the caller formats on the host). With `null_value` (tplx_gpu_result_csv_nulls) a None cell of
        an Option[T] column is written as that value, quoted once; without it a result with Option[T] columns returns None."""
        def call(buf, n, need):
            if null_value is None:
                return lib().tplx_gpu_result_csv(self._h, n_cols, ord(delimiter), ord(quotechar), buf, n, ct.byref(need))
            return lib().tplx_gpu_result_csv_nulls(self._h, n_cols, ord(delimiter), ord(quotechar), null_value.encode(), buf, n,
                                                   ct.byref(need))
        need = ct.c_uint64()
        rc = call(None, 0, need)
        if rc == -6:  # TPLX_E_UNSUPPORTED
            return None
        _check(rc, "tplx_gpu_result_csv")
        buf = np.empty(need.value, dtype=np.uint8)
        if need.value:
            _check(call(buf.ctypes.data, need.value, need), "tplx_gpu_result_csv")
        return buf.tobytes()

    def merge_resolved(self, resolved: "Block", row_nos: Sequence[int], first_row_no: int = 0) -> "Result":
        """In-order merge of resolved rows on the device (K9, tplx_gpu_result_merge_resolved; ResolveTask::executeInOrder):
        `resolved` holds the stage's visible output columns, one row per resolved exception, ordered by row number."""
        arr = (ct.c_int64 * max(len(row_nos), 1))(*[int(v) for v in row_nos])
        h = ct.c_void_p()
        _check(lib().tplx_gpu_result_merge_resolved(self._h, resolved._h, arr, first_row_no, ct.byref(h)), "tplx_gpu_result_merge_resolved")
        r = Result(h, None, resolved, types=self.out_types())
        r._rowidx = self.rowidx
        return r

    def sort_by_keys(self, n_keys: int, col_flags: Optional[Sequence[int]] = None) -> "Result":
        """The rows ordered by the first `n_keys` columns, stably, None first (K11, tplx_gpu_result_sort_by_keys), as a new result
        with the same visible columns; `col_flags` holds 0 or CONCAT_DROP_VALID per column (None: 0 for every column)."""
        h = ct.c_void_p()
        flags = bytes(col_flags) if col_flags is not None else None
        _check(lib().tplx_gpu_result_sort_by_keys(self._h, n_keys, flags, ct.byref(h)), "tplx_gpu_result_sort_by_keys")
        r = Result(h, None, None, types=self.out_types())
        r._rowidx = self.rowidx
        r.device = self.device
        return r

    def exception_partition(self) -> bytes:
        need = ct.c_uint64()
        _check(lib().tplx_gpu_result_exception_partition(self._h, None, 0, ct.byref(need)), "result_exception_partition(size)")
        buf = np.empty(need.value, dtype=np.uint8)
        _check(lib().tplx_gpu_result_exception_partition(self._h, buf.ctypes.data, buf.nbytes, ct.byref(need)),
               "result_exception_partition")
        return buf.tobytes()

    def free(self):
        if self._h:
            lib().tplx_gpu_result_free(self._h)
            self._h = ct.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------------
# hash join (K8): build once, probe block after block
# ------------------------------------------------------------------------------------------------
JOIN_LEFT_OUTER = ir.C["TPLX_JOIN_LEFT_OUTER"]
JOIN_BUILD_FIRST = ir.C["TPLX_JOIN_BUILD_FIRST"]


class Join:
    """Device hash table over one key column of the build side (tplx_gpu_join_build); replaces the reference's build stage with a
    hash-table endpoint (TransformTask.cc:769-842). probe() = the hash-join probe of the row pipeline (PipelineBuilder.cc:2110-2523)."""

    def __init__(self, build: Block, build_types: Sequence[int], key_col: int):
        self.build = build  # borrowed by the table: keep it alive
        self.build_types = list(build_types)
        self.key_col = key_col
        self._h = ct.c_void_p()
        _check(lib().tplx_gpu_join_build(build._h, key_col, ct.byref(self._h)), "tplx_gpu_join_build")

    @property
    def info(self):
        n, nn, ms, kl = ct.c_uint64(), ct.c_uint64(), ct.c_double(), ct.c_uint32()
        _check(lib().tplx_gpu_join_info(self._h, ct.byref(n), ct.byref(nn), ct.byref(ms), ct.byref(kl)), "tplx_gpu_join_info")
        return {"n_rows": n.value, "n_null_rows": nn.value, "build_ms": ms.value, "kernel_launches": kl.value}

    def out_types(self, probe_types: Sequence[int], probe_key: int, build_first: bool) -> List[int]:
        pt = [t for i, t in enumerate(probe_types) if i != probe_key]
        bt = [t for i, t in enumerate(self.build_types) if i != self.key_col]
        kt = [probe_types[probe_key]]
        return bt + kt + pt if build_first else pt + kt + bt

    def probe(self, probe: Block, probe_types: Sequence[int], probe_key: int, left_outer: bool = False, build_first: bool = False) -> Result:
        h = ct.c_void_p()
        flags = (JOIN_LEFT_OUTER if left_outer else 0) | (JOIN_BUILD_FIRST if build_first else 0)
        _check(lib().tplx_gpu_join_probe(self._h, probe._h, probe_key, flags, ct.byref(h)), "tplx_gpu_join_probe")
        return Result(h, None, probe, types=self.out_types(probe_types, probe_key, build_first))

    def free(self):
        if self._h:
            lib().tplx_gpu_join_destroy(self._h)
            self._h = ct.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------------
# CSV source (K6): bytes -> column block on the device
# ------------------------------------------------------------------------------------------------
class CsvBuffer:
    """CSV text resident on a device (tplx_gpu_csv_upload)."""

    def __init__(self, device: int, data):
        init([device])
        self.device = device
        self._arr = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        self.n_bytes = int(self._arr.size)
        self._h = ct.c_void_p()
        _check(lib().tplx_gpu_csv_upload(device, self._arr.ctypes.data if self.n_bytes else None, self.n_bytes, ct.byref(self._h)),
               "tplx_gpu_csv_upload")

    def parse(self, col_types: Sequence[int], delimiter=",", quotechar='"', header=False, null_values: Sequence[str] = ("",),
              lazy: Optional[Sequence[int]] = None) -> "CsvParse":
        """lazy: file-column indices of string columns that stay as cell references (materialised by Stage.run only for the
        rows its prefilter lets through); the buffer must stay alive as long as the block."""
        d = CCsvDesc()
        d.delimiter, d.quotechar, d.skip_header = ord(delimiter), ord(quotechar), int(bool(header))
        d.n_null_values = len(null_values)
        d.n_file_cols = len(col_types)
        types = bytes(col_types)
        d.col_types = types
        nv = (ct.c_char_p * max(1, len(null_values)))(*[s.encode() for s in null_values])
        d.null_values = nv
        lz = bytes(1 if (lazy and c in lazy) else 0 for c in range(len(col_types)))
        d.col_lazy = lz if lazy else None
        hb, hr = ct.c_void_p(), ct.c_void_p()
        _check(lib().tplx_gpu_csv_parse(self._h, ct.byref(d), ct.byref(hb), ct.byref(hr)), "tplx_gpu_csv_parse")
        nr = ct.c_uint64()
        _check(lib().tplx_gpu_block_rows(hb, ct.byref(nr)), "tplx_gpu_block_rows")
        return CsvParse(Block(hb, nr.value, self.device), hr, [t for t in col_types if t != CSV_SKIP])

    def parse_text(self, null_values: Sequence[str] = (), option: bool = False) -> "CsvParse":
        """K10 (tplx_gpu_text_parse): every line one row of a single string column. A line equal to a null value is None with
        `option` (Option[str] column), else a bad row (NULLERROR) for the interpreter path."""
        d = CTextDesc()
        d.n_null_values = len(null_values)
        d.option = int(bool(option))
        nv = (ct.c_char_p * max(1, len(null_values)))(*[s.encode() for s in null_values])
        d.null_values = nv
        hb, hr = ct.c_void_p(), ct.c_void_p()
        _check(lib().tplx_gpu_text_parse(self._h, ct.byref(d), ct.byref(hb), ct.byref(hr)), "tplx_gpu_text_parse")
        nr = ct.c_uint64()
        _check(lib().tplx_gpu_block_rows(hb, ct.byref(nr)), "tplx_gpu_block_rows")
        return CsvParse(Block(hb, nr.value, self.device), hr, [T_STR])

    def free(self):
        if self._h:
            lib().tplx_gpu_csv_buffer_free(self._h)
            self._h = ct.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class CsvParse:
    """Result of CsvBuffer.parse: `.block` feeds Stage.run; bad rows go to the interpreter path."""

    def __init__(self, block: Block, h, types: List[int]):
        self.block, self._h, self.types = block, h, types
        self._info = None

    @property
    def info(self) -> CCsvInfo:
        if self._info is None:
            i = CCsvInfo()
            _check(lib().tplx_gpu_csv_result_info(self._h, ct.byref(i)), "tplx_gpu_csv_result_info")
            self._info = i
        return self._info

    def bad_rows(self) -> np.ndarray:
        out = np.zeros(int(self.info.n_bad), dtype=CSV_BAD_DTYPE)
        _check(lib().tplx_gpu_csv_result_fetch_bad_rows(self._h, out.ctypes.data if len(out) else None), "tplx_gpu_csv_result_fetch_bad_rows")
        return out

    def rowmap(self) -> np.ndarray:
        out = np.zeros(int(self.info.n_normal), dtype=np.uint32)
        _check(lib().tplx_gpu_csv_result_fetch_rowmap(self._h, out.ctypes.data if len(out) else None), "tplx_gpu_csv_result_fetch_rowmap")
        return out

    def block_bytes(self) -> List[int]:
        """bytes of every column of the parsed block (values, or string payload + offsets)"""
        arr = (ct.c_uint64 * 64)()
        n = ct.c_uint32()
        _check(lib().tplx_gpu_block_column_bytes(self.block._h, arr, 64, ct.byref(n)), "tplx_gpu_block_column_bytes")
        return [int(arr[i]) for i in range(n.value)]

    def row_ends(self) -> np.ndarray:
        """ends[i] + 1 .. ends[i + 1]: byte window of data row i (leading newlines to be skipped); ends[0] wraps to -1."""
        out = np.zeros(int(self.info.n_rows) + 1, dtype=np.uint32)
        _check(lib().tplx_gpu_csv_result_fetch_row_ends(self._h, out.ctypes.data), "tplx_gpu_csv_result_fetch_row_ends")
        return out

    def free(self):
        if self._h:
            lib().tplx_gpu_csv_result_free(self._h)
            self._h = ct.c_void_p()
        self.block.free()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
