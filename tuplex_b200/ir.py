"""Stage descriptor ("op program") builder — Python mirror of include/tplx_ir.h.

The enumerators are parsed out of the C header at import time so the two sides cannot drift.
A reference TransformStage carries LLVM bitcode (tuplex/core/src/physical/StageBuilder.cc:1499-1535);
ours carries this flat predicated register program instead.
"""
from __future__ import annotations

import os
import re
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

_HDR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "tplx_ir.h")


def _parse_header(path: str) -> Dict[str, int]:
    txt = open(path).read()
    consts: Dict[str, int] = {}
    for m in re.finditer(r"^\s*(TPLX_[A-Z0-9_]+)\s*=\s*(-?\d+)\s*,", txt, re.M):
        consts[m.group(1)] = int(m.group(2))
    for m in re.finditer(r"^#define\s+(TPLX_[A-Z0-9_]+)\s+(0x[0-9A-Fa-f]+|\d+)u?\s*(?:/\*.*)?$", txt, re.M):
        consts[m.group(1)] = int(m.group(2), 0)
    return consts


C = _parse_header(_HDR)
C.update({k: v for k, v in _parse_header(os.path.join(os.path.dirname(_HDR), "tplx_gpu.h")).items() if k == "TPLX_COMM_ID_BYTES" or k.startswith("TPLX_JOIN_")})
globals().update(C)  # TPLX_OP_*, TPLX_T_*, ... become module attributes

T_I64, T_F64, T_BOOL, T_STR = C["TPLX_T_I64"], C["TPLX_T_F64"], C["TPLX_T_BOOL"], C["TPLX_T_STR"]
TYPE_NAMES = {T_I64: "i64", T_F64: "f64", T_BOOL: "bool", T_STR: "str"}
NOSLOT = C["TPLX_NOSLOT"]
OP_NAMES = {v: k[len("TPLX_OP_"):] for k, v in C.items() if k.startswith("TPLX_OP_")}

INSTR_FMT = "<BBHHHHHHHqq"  # 32 bytes
assert struct.calcsize(INSTR_FMT) == 32
HEADER_FMT = "<IIIHHHHHHIIBBHIII"
assert struct.calcsize(HEADER_FMT) == 48


@dataclass
class Instr:
    op: int
    dst: int = NOSLOT
    a: int = NOSLOT
    b: int = NOSLOT
    c: int = NOSLOT
    guard: int = NOSLOT
    opidx: int = 0
    flags: int = 0
    imm: int = 0
    imm2: int = 0

    def pack(self) -> bytes:
        return struct.pack(INSTR_FMT, self.op, self.flags, self.dst, self.a, self.b, self.c, self.guard,
                           self.opidx, 0, _as_i64(self.imm), _as_i64(self.imm2))

    def __repr__(self):
        return (f"{OP_NAMES.get(self.op, self.op)} dst={self.dst} a={self.a} b={self.b} c={self.c} "
                f"g={self.guard} fl={self.flags} imm={self.imm} imm2={self.imm2} op#{self.opidx}")


@dataclass
class Acc:
    kind: int
    slot: int
    init_bits: int  # raw 64-bit pattern (i64 value or f64 bits)


@dataclass
class Program:
    """A complete stage: input schema, instructions, output row / accumulators / keys."""
    in_types: List[int]
    in_names: List[Optional[str]]
    instrs: List[Instr] = field(default_factory=list)
    cpool: bytearray = field(default_factory=bytearray)
    out_cols: List[Tuple[int, int]] = field(default_factory=list)  # (slot, type)
    out_names: List[Optional[str]] = field(default_factory=list)
    accs: List[Acc] = field(default_factory=list)
    n_keys: int = 0
    opids: List[int] = field(default_factory=list)
    n_slots: int = 0
    endpoint: int = 0
    hidden_out_cols: int = 0
    null_of: Dict[int, int] = field(default_factory=dict)   # input column j is the "is None" companion of Option[T] input column null_of[j]
    out_null_of: List[int] = field(default_factory=list)    # per output column: 0, or 1 + the output column it is the "is None" companion of
    prefilter: Optional["Program"] = None  # selective leading part, output = surviving row indices
    fused: Optional[bytes] = None  # serialized tplx_fused_header section (closed-form scan-aggregate hint)
    scratch_bytes: int = 256
    _cpool_index: Dict[bytes, int] = field(default_factory=dict)

    def const_bytes(self, b: bytes) -> Tuple[int, int]:
        if b in self._cpool_index:
            return self._cpool_index[b], len(b)
        off = len(self.cpool)
        self.cpool += b
        # keep constants 8-byte separated so that views never alias by accident
        while len(self.cpool) % 8:
            self.cpool.append(0)
        self._cpool_index[b] = off
        return off, len(b)

    def serialize(self) -> bytes:
        def pad8(b: bytes) -> bytes:
            return b + b"\0" * ((-len(b)) % 8)

        body = b""
        body += pad8(bytes((C["TPLX_T_NULLOF"] | self.null_of[j]) if j in self.null_of else t for j, t in enumerate(self.in_types)))
        nof = list(self.out_null_of) + [0] * (len(self.out_cols) - len(self.out_null_of))
        body += pad8(b"".join(struct.pack("<HBB", s, t, nof[k]) for k, (s, t) in enumerate(self.out_cols)))
        body += b"".join(struct.pack("<BBHIq", a.kind, 0, a.slot, 0, _as_i64(a.init_bits)) for a in self.accs)
        body += b"".join(struct.pack("<q", o) for o in self.opids)
        body += b"".join(i.pack() for i in self.instrs)
        body += pad8(bytes(self.cpool))
        pre = self.prefilter.serialize() if self.prefilter is not None else b""
        body += pre
        fused = self.fused or b""
        body += fused
        total = struct.calcsize(HEADER_FMT) + len(body)
        hdr = struct.pack(HEADER_FMT, C["TPLX_IR_MAGIC"], C["TPLX_IR_VERSION"], total, len(self.in_types),
                          len(self.out_cols), len(self.accs), self.n_keys, len(self.opids), self.n_slots,
                          len(self.instrs), len(self.cpool), self.endpoint, 0, self.hidden_out_cols, self.scratch_bytes,
                          len(pre), len(fused))
        return hdr + body

    def dump(self) -> str:
        lines = [f"in: {[TYPE_NAMES[t] for t in self.in_types]} slots={self.n_slots} prefilter={self.prefilter is not None}"]
        for i, ins in enumerate(self.instrs):
            lines.append(f"{i:4d}: {ins!r}")
        lines.append(f"out: {[(s, TYPE_NAMES[t]) for s, t in self.out_cols]} accs={self.accs} keys={self.n_keys}")
        return "\n".join(lines)


def _as_i64(bits: int) -> int:
    bits &= (1 << 64) - 1
    return bits - (1 << 64) if bits >= 1 << 63 else bits


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b & ((1 << 64) - 1)))[0]


SCAN_HDR_FMT = "<IIQ"              # tplx_scan_header
SCAN_TERM_FMT = "<IIIIqQQqIIQ"      # tplx_scan_term (64 bytes)
assert struct.calcsize(SCAN_TERM_FMT) == 64 and struct.calcsize(SCAN_HDR_FMT) == 16


def scan_terms(blob: Optional[bytes]) -> Optional[List[dict]]:
    """Decode a string-scan hint (tplx_scan_header + terms); None when blob is not one."""
    if not blob or len(blob) < 16:
        return None
    magic, n, _ = struct.unpack_from(SCAN_HDR_FMT, blob, 0)
    if magic != C["TPLX_SCAN_MAGIC"]:
        return None
    keys = ("kind", "col", "flags", "cmp", "imm", "needle", "sep", "skip", "opidx_val", "opidx_filter", "pad")
    return [dict(zip(keys, struct.unpack_from(SCAN_TERM_FMT, blob, 16 + 64 * i))) for i in range(n)]


def pack_scan_terms(terms: List[dict]) -> bytes:
    out = struct.pack(SCAN_HDR_FMT, C["TPLX_SCAN_MAGIC"], len(terms), 0)
    for t in terms:
        out += struct.pack(SCAN_TERM_FMT, t["kind"], t["col"], t["flags"], t.get("cmp", 0), _as_i64(t.get("imm", 0)), t.get("needle", 0),
                           t.get("sep", 0), _as_i64(t.get("skip", 0)), t.get("opidx_val", 0), t.get("opidx_filter", 0), 0)
    return out


def referenced_inputs(prog: Program) -> List[int]:
    """Physical input columns a stage actually loads (projection pushdown: the reference keeps only these when it reads a
    file, LogicalOptimizer projection pushdown / `columnsToSerialize`, StageBuilder.cc:1045-1070). A load of an "is None"
    companion counts as a use of its Option[T] column, whose validity bitmap fills the companion."""
    used = set()
    p = prog
    while p is not None:
        used.update(p.null_of.get(int(i.imm), int(i.imm)) for i in p.instrs if i.op == C["TPLX_OP_LDCOL"])
        p = p.prefilter
    if prog.fused and scan_terms(prog.fused) is None:
        _, n_preds, n_terms, _ = struct.unpack_from("<IIII", prog.fused, 0)
        off = 16
        for _ in range(n_preds):
            used.add(struct.unpack_from("<I", prog.fused, off)[0])
            off += 24
        for _ in range(n_terms):
            _, op, ca, cb = struct.unpack_from("<IIII", prog.fused, off)
            if op in (C["TPLX_FT_COL"], C["TPLX_FT_MUL"]):
                used.add(ca)
            if op == C["TPLX_FT_MUL"]:
                used.add(cb)
            off += 32
    return sorted(used)


def project_inputs(prog: Program, used: List[int]) -> None:
    """Renumber the input columns of `prog` (in place) so that it reads a block holding only the physical columns `used`. The
    companion of every projected Option[T] column follows them, in the order of its column, where the executor appends the
    companions (tplx_gpu_stage_run); companions of columns left out are dropped."""
    remap = {c: k for k, c in enumerate(used)}
    p = prog
    while p is not None:
        comps = sorted((c, j) for j, c in p.null_of.items() if c in remap)
        cmap = {j: len(used) + m for m, (_, j) in enumerate(comps)}
        for i in p.instrs:
            if i.op == C["TPLX_OP_LDCOL"]:
                i.imm = cmap[int(i.imm)] if int(i.imm) in p.null_of else remap[int(i.imm)]
        keep = list(used) + [j for _, j in comps]
        p.in_types = [p.in_types[c] for c in keep]
        p.in_names = [p.in_names[c] for c in keep] if p.in_names else p.in_names
        p.null_of = {cmap[j]: remap[c] for c, j in comps}
        terms = scan_terms(p.fused)
        if terms is not None:  # string-scan hint of a (prefilter) row stage: its terms name input columns too
            for t in terms:
                t["col"] = remap[t["col"]]
            p.fused = pack_scan_terms(terms)
        p = p.prefilter
    if prog.fused and scan_terms(prog.fused) is None:
        b = bytearray(prog.fused)
        _, n_preds, n_terms, _ = struct.unpack_from("<IIII", b, 0)
        off = 16
        for _ in range(n_preds):
            struct.pack_into("<I", b, off, remap[struct.unpack_from("<I", b, off)[0]])
            off += 24
        for _ in range(n_terms):
            _, op, ca, cb = struct.unpack_from("<IIII", b, off)
            if op in (C["TPLX_FT_COL"], C["TPLX_FT_MUL"]):
                struct.pack_into("<I", b, off + 8, remap[ca])
            if op == C["TPLX_FT_MUL"]:
                struct.pack_into("<I", b, off + 12, remap[cb])
            off += 32
        prog.fused = bytes(b)
