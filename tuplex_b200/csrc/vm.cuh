// vm.cuh — per-row evaluator of the tplx op program on sm_90a.
//
// Replaces the body of the LLVM-generated processRow pipeline
// (reference tuplex/core/src/physical/PipelineBuilder.cc:90-170,565-1025) and the UDF code that
// BlockGeneratorVisitor/FunctionRegistry emit. One thread evaluates one row at a time; the
// program is warp-uniform, so decode is uniform and only the data path diverges.
// The register file lives in shared memory as regs[slot][thread] (8-byte slots; bank-conflict
// free because consecutive threads touch consecutive 8-byte words).
//
// The host pre-decodes tplx_instr (include/tplx_ir.h) into DInstr: slot numbers become byte offsets into
// the register file, op/flags/operator-index are packed into one word, so that dispatch is
// a few 128-bit broadcast loads + one jump-table branch.
//
// Semantics cited per op in include/tplx_ir.h; the CPU restatement that this file must match
// bit-for-bit is oracle/tplx_oracle.c.
#pragma once
#include <stdint.h>
#include "../../include/tplx_ir.h"
#include "strops.cuh"
#include "csvops.cuh"

namespace tplx {

constexpr uint32_t NOOFF = 0xFFFFFFFFu;

struct __align__(16) DInstr {
    uint32_t op_flags;  // op | flags << 8 | opidx << 16
    uint32_t dst, a, b; // byte offsets of slots inside a thread's register column (slot * NT * 8), NOOFF = none
    uint32_t c, guard, pad0, pad1;
    int64_t imm, imm2;
};
static_assert(sizeof(DInstr) == 48, "DInstr layout");

struct VMThread {
    bool alive;          // row still in the pipeline (valid, not filtered, no exception)
    uint32_t exc_code;   // 0 = none
    uint32_t exc_op;     // operator index of the raising op
    uint8_t *scratch;    // per-thread arena for materialised strings
    uint32_t scr_used;
    uint32_t scr_cap;
};

struct ColIn {
    const void *data;
    const uint32_t *offsets;
    uint64_t type;
};

// float(str): out of line so that the VM's register allocation is not shaped by a rarely used op
TPLX_HD_NOINLINE bool str_to_f64(StrV s, double *out) {
    return csv_atod_g([&s](uint32_t k) { return sch(s, k); }, s.len, out);
}

__device__ __forceinline__ uint8_t *scratch_alloc(VMThread &t, uint32_t n, uint32_t opidx) {
    if (t.scr_used + n > t.scr_cap) {
        // internal limit, not a Python error: hand the row to the resolve path
        t.exc_code = TPLX_EC_NORMALCASEVIOLATION;
        t.exc_op = opidx;
        t.alive = false;
        return nullptr;
    }
    uint8_t *p = t.scratch + t.scr_used;
    t.scr_used += n;
    return p;
}

__device__ __forceinline__ void raise_exc(VMThread &t, uint32_t code, uint32_t opidx) {
    t.exc_code = code;
    t.exc_op = opidx;
    t.alive = false;
}

// ---- op bodies shared by the interpreter (VM::run below) and the stage specialiser's generated code (jit.inl): one
// implementation of every non-trivial op, written on plain values (StrV views, integers), not on the register file ---------------
#ifdef TPLX_JIT
#define TPLX_OPFN_HEAVY __device__ __noinline__   // generated code may use an op several times: one out-of-line copy
#else
#define TPLX_OPFN_HEAVY __device__ __forceinline__
#endif
__device__ __forceinline__ bool op_icmp(uint32_t pred, int64_t x, int64_t y) {
    switch (pred) {
        case TPLX_CMP_EQ: return x == y;
        case TPLX_CMP_NE: return x != y;
        case TPLX_CMP_LT: return x < y;
        case TPLX_CMP_LE: return x <= y;
        case TPLX_CMP_GT: return x > y;
        default: return x >= y;
    }
}
__device__ __forceinline__ bool op_fcmp(uint32_t pred, double x, double y) {  // ordered predicates: false if either is NaN
    switch (pred) {
        case TPLX_CMP_EQ: return x == y;
        case TPLX_CMP_NE: return (x < y) || (x > y);  // FCMP_ONE
        case TPLX_CMP_LT: return x < y;
        case TPLX_CMP_LE: return x <= y;
        case TPLX_CMP_GT: return x > y;
        default: return x >= y;
    }
}
__device__ __forceinline__ double op_fmod(double x, double y) {  // y != 0
    double r = fmod(x, y);  // == LLVM frem, exact
    if (r != 0.0 && ((r < 0.0) != (y < 0.0))) r = __dadd_rn(r, y);
    return r;
}
__device__ __forceinline__ StrV mk_strv(const uint8_t *p, uint32_t len, uint32_t flags) {
    StrV v;
    v.p = p;
    v.len = len;
    v.flags = flags;
    return v;
}
__device__ __forceinline__ bool op_sstarts(const StrV &s, const StrV &p) {
    bool r = p.len <= s.len;
    for (uint32_t i = 0; r && i < p.len; ++i) r = sch(s, i) == sch(p, i);
    return r;
}
__device__ __forceinline__ bool op_sends(const StrV &s, const StrV &p) {
    bool r = p.len <= s.len;
    for (uint32_t i = 0; r && i < p.len; ++i) r = sch(s, s.len - p.len + i) == sch(p, i);
    return r;
}
__device__ __forceinline__ StrV op_sslice(const StrV &s, uint32_t flags, int64_t b, int64_t c) {
    const int64_t len = s.len;
    const int64_t st = (flags & TPLX_SL_HAS_START) ? slice_index(b, len) : 0;
    const int64_t en = (flags & TPLX_SL_HAS_END) ? slice_index(c, len) : len;
    if (st < en) return mk_strv(s.p + st, (uint32_t)(en - st), s.flags);
    return mk_strv(s.p, 0, 0);
}
__device__ __forceinline__ bool op_sindex(const StrV &s, int64_t idx, StrV *out) {  // false = IndexError
    if (idx < 0) idx += s.len;
    if (idx < 0 || idx >= (int64_t)s.len) return false;
    *out = mk_strv(s.p + idx, 1, s.flags);
    return true;
}
__device__ __forceinline__ StrV op_sstrip(const StrV &s, uint32_t flags) {
    uint32_t i = 0, e = s.len;
    if (flags & 1) while (i < e && is_pyspace(s.p[i])) ++i;
    if (flags & 2) while (e > i && is_pyspace(s.p[e - 1])) --e;
    return mk_strv(s.p + i, e - i, s.flags);
}
// the materialising ops return false when the per-row scratch arena is exhausted (the row has been marked by scratch_alloc)
__device__ __forceinline__ bool op_sconcat(VMThread &t, const StrV &x, const StrV &y, uint32_t opidx, StrV *out) {
    // empty operand returns the other side unchanged (BlockGeneratorVisitor.cc:381-436)
    if (x.len == 0) { *out = y; return true; }
    if (y.len == 0) { *out = x; return true; }
    uint8_t *o = scratch_alloc(t, x.len + y.len, opidx);
    if (!o) return false;
    str_copy(o, x);
    str_copy(o + x.len, y);
    *out = mk_strv(o, x.len + y.len, 0);
    return true;
}
TPLX_OPFN_HEAVY bool op_sreplace(VMThread &t, StrV s, StrV f, StrV r, uint32_t opidx, StrV *out) {
    // runtime/src/Runtime.cc:401-540
    if (s.len == 0 || (f.len == 0 && r.len == 0)) { *out = s; return true; }
    if (f.len == 0) {
        uint32_t n = (r.len + 1) * s.len + r.len;
        uint8_t *o = scratch_alloc(t, n, opidx);
        if (!o) return false;
        uint32_t pos = 0;
        for (uint32_t i = 0; i < s.len; ++i) {
            for (uint32_t j = 0; j < r.len; ++j) o[pos++] = sch(r, j);
            o[pos++] = sch(s, i);
        }
        for (uint32_t j = 0; j < r.len; ++j) o[pos++] = sch(r, j);
        *out = mk_strv(o, pos, 0);
        return true;
    }
    if (f.len == 1 && s.flags == TPLX_SF_NONE && f.flags == TPLX_SF_NONE && r.flags == TPLX_SF_NONE) {
        // single-character needle on a plain string (the common `.replace(',', '')`): two byte loops without case mapping
        const uint8_t ch = f.p[0];
        uint32_t cnt = 0;
        for (uint32_t q = 0; q < s.len; ++q) cnt += s.p[q] == ch;
        if (cnt == 0) { *out = mk_strv(s.p, s.len, 0); return true; }  // nothing to replace: the input itself (same bytes as a copy)
        const uint32_t n1 = s.len + cnt * r.len - cnt;
        uint8_t *o1 = scratch_alloc(t, n1 ? n1 : 1, opidx);
        if (!o1) return false;
        uint32_t w = 0;
        for (uint32_t q = 0; q < s.len; ++q) {
            const uint8_t b0 = s.p[q];
            if (b0 == ch) for (uint32_t j = 0; j < r.len; ++j) o1[w++] = r.p[j];
            else o1[w++] = b0;
        }
        *out = mk_strv(o1, n1, 0);
        return true;
    }
    // count pass
    uint32_t count = 0, i = 0;
    while (i + f.len <= s.len) {
        uint32_t j = 0;
        while (j < f.len && sch(s, i + j) == sch(f, j)) ++j;
        if (j == f.len) { ++count; i += f.len; } else ++i;
    }
    if (count == 0) { *out = s; return true; }  // nothing to replace: the input itself, like the single-character path
    uint32_t n = s.len + count * r.len - count * f.len;
    uint8_t *o = scratch_alloc(t, n ? n : 1, opidx);
    if (!o) return false;
    uint32_t pos = 0;
    i = 0;
    while (i < s.len) {
        bool m = false;
        if (i + f.len <= s.len) {
            uint32_t j = 0;
            while (j < f.len && sch(s, i + j) == sch(f, j)) ++j;
            m = (j == f.len);
        }
        if (m) {
            for (uint32_t j = 0; j < r.len; ++j) o[pos++] = sch(r, j);
            i += f.len;
        } else o[pos++] = sch(s, i++);
    }
    *out = mk_strv(o, pos, 0);
    return true;
}
TPLX_OPFN_HEAVY bool op_sfmtd(VMThread &t, uint32_t flags, uint64_t raw, uint32_t width, uint32_t opidx, StrV *out) {
    // '%[0]<w>d' % v: snprintf with C's %d, which consumes an int (BlockGeneratorVisitor.cc:675-775);
    // flags bit1: '{:0<w>}'.format(v) / f-strings go through fmt and keep all 64 bits (Runtime.cc:544-607)
    const int64_t v = (flags & 2) ? (int64_t)raw : (int64_t)(int32_t)(int64_t)raw;
    uint64_t mag = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    uint32_t nd = 1;
    for (uint64_t q = mag; q >= 10; q /= 10) ++nd;
    uint32_t body = nd + (v < 0 ? 1 : 0);
    uint32_t total = body > width ? body : width;
    uint8_t *o = scratch_alloc(t, total, opidx);
    if (!o) return false;
    uint32_t padn = total - body, pos = 0;
    if (flags & 1) {
        if (v < 0) o[pos++] = '-';
        for (uint32_t i = 0; i < padn; ++i) o[pos++] = '0';
    } else {
        for (uint32_t i = 0; i < padn; ++i) o[pos++] = ' ';
        if (v < 0) o[pos++] = '-';
    }
    for (uint32_t i = 0; i < nd; ++i) { o[pos + nd - 1 - i] = (uint8_t)('0' + mag % 10); mag /= 10; }
    *out = mk_strv(o, total, 0);
    return true;
}
TPLX_OPFN_HEAVY bool op_i2s(VMThread &t, int64_t v, uint32_t opidx, StrV *out) {
    uint64_t mag = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    uint32_t nd = 1;
    for (uint64_t q = mag; q >= 10; q /= 10) ++nd;
    uint32_t total = nd + (v < 0 ? 1 : 0);
    uint8_t *o = scratch_alloc(t, total, opidx);
    if (!o) return false;
    if (v < 0) o[0] = '-';
    for (uint32_t i = 0; i < nd; ++i) { o[total - 1 - i] = (uint8_t)('0' + mag % 10); mag /= 10; }
    *out = mk_strv(o, total, 0);
    return true;
}

template <int NT>
struct VM {
    static constexpr uint32_t SLOT_BYTES = NT * 8;  // distance between consecutive slots of one thread

    // rb = this thread's register column (byte pointer); off = slot byte offset
    static __device__ __forceinline__ uint64_t &R(uint8_t *rb, uint32_t off) { return *reinterpret_cast<uint64_t *>(rb + off); }
    static __device__ __forceinline__ StrV RS(uint8_t *rb, uint32_t off) {
        StrV v;
        v.p = (const uint8_t *)R(rb, off);
        uint64_t m = R(rb, off + SLOT_BYTES);
        v.len = (uint32_t)m;
        v.flags = (uint32_t)(m >> 32);
        return v;
    }
    static __device__ __forceinline__ void WS(uint8_t *rb, uint32_t off, const uint8_t *p, uint32_t len, uint32_t flags) {
        R(rb, off) = (uint64_t)p;
        R(rb, off + SLOT_BYTES) = (uint64_t)len | ((uint64_t)flags << 32);
    }
    static __device__ __forceinline__ StrV CS(const uint8_t *cpool, int64_t enc) {  // constant-pool view
        StrV v;
        v.p = cpool + (uint32_t)enc;
        v.len = (uint32_t)((uint64_t)enc >> 32);
        v.flags = 0;
        return v;
    }

    // Run instructions [pc0, pc1) for this thread's row.
    // row = input row index (LDROW, exceptions); w = position in the work list (== row unless a row list is used):
    // columns flagged compact (gather.cuh) are indexed by w.
    static __device__ void run(const DInstr *__restrict__ prog, uint32_t pc0, uint32_t pc1, uint8_t *__restrict__ rb,
                               const ColIn *__restrict__ cols, uint64_t row, uint64_t w, const uint8_t *__restrict__ cpool, VMThread &t) {
        bool check_alive = false;
        for (uint32_t pc = pc0; pc < pc1; ++pc) {
            // uniform fetch (broadcast from shared memory)
            const uint4 w0 = *reinterpret_cast<const uint4 *>(&prog[pc]);
            const uint2 w1 = *reinterpret_cast<const uint2 *>(&prog[pc].c);
            const uint32_t op = w0.x & 0xFF;
            const uint32_t flags = (w0.x >> 8) & 0xFF;
            const uint32_t opidx = w0.x >> 16;
            const uint32_t dst = w0.y, a = w0.z, b = w0.w, c = w1.x, guard = w1.y;
            bool act = t.alive;
            if (guard != NOOFF) {
                act = act && (R(rb, guard) != 0);
                if (!__any_sync(0xFFFFFFFFu, act)) continue;  // untaken branch of an if-converted UDF: whole warp skips the op
            } else if (check_alive) {
                // the previous instruction was a FILTER: when it emptied the warp nothing that follows can execute
                if (!__any_sync(0xFFFFFFFFu, act)) return;
            }
            check_alive = op == TPLX_OP_FILTER;  // warp-uniform
            if (!act) continue;
            const int64_t imm = prog[pc].imm;
            // operand fetch (constant operands come from the immediates: a <- imm2, b <- imm, c <- imm2)
#define IA() ((flags & TPLX_F_A_CONST) ? (uint64_t)prog[pc].imm2 : R(rb, a))
#define IB() ((flags & TPLX_F_B_CONST) ? (uint64_t)imm : R(rb, b))
#define IC() ((flags & TPLX_F_C_CONST) ? (uint64_t)prog[pc].imm2 : R(rb, c))
#define FA() __longlong_as_double((long long)IA())
#define FB() __longlong_as_double((long long)IB())
#define SA() ((flags & TPLX_F_A_CONST) ? CS(cpool, prog[pc].imm2) : RS(rb, a))
#define SB() ((flags & TPLX_F_B_CONST) ? CS(cpool, imm) : RS(rb, b))
#define SC() ((flags & TPLX_F_C_CONST) ? CS(cpool, prog[pc].imm2) : RS(rb, c))
#define WF(x) R(rb, dst) = (uint64_t)__double_as_longlong(x)
            switch (op) {
                case TPLX_OP_LDCOL: {
                    const ColIn &ci = cols[imm];
                    const uint64_t idx = (ci.type & 0x100) ? w : row;  // COL_COMPACT
                    if (flags == TPLX_T_STR) {
                        uint32_t o0 = ci.offsets[idx], o1 = ci.offsets[idx + 1];
                        WS(rb, dst, (const uint8_t *)ci.data + o0, o1 - o0, 0);
                    } else {
                        R(rb, dst) = ((const uint64_t *)ci.data)[idx];
                    }
                    break;
                }
                case TPLX_OP_LDI: R(rb, dst) = (uint64_t)imm; break;
                case TPLX_OP_LDROW: R(rb, dst) = row; break;
                case TPLX_OP_LDS: {
                    StrV s = CS(cpool, imm);
                    WS(rb, dst, s.p, s.len, 0);
                    break;
                }
                case TPLX_OP_MOV:
                    if ((flags & 3) == 2) {
                        StrV s = SA();
                        WS(rb, dst, s.p, s.len, s.flags);
                    } else R(rb, dst) = IA();
                    break;
                case TPLX_OP_SEL: {
                    const bool pick_a = R(rb, c) != 0;
                    if ((flags & 3) == 2) {
                        StrV s = pick_a ? SA() : SB();
                        WS(rb, dst, s.p, s.len, s.flags);
                    } else R(rb, dst) = pick_a ? IA() : IB();
                    break;
                }
                case TPLX_OP_IADD: R(rb, dst) = IA() + IB(); break;
                case TPLX_OP_ISUB: R(rb, dst) = IA() - IB(); break;
                case TPLX_OP_IMUL: R(rb, dst) = IA() * IB(); break;
                case TPLX_OP_IFLOORDIV: {
                    int64_t y = (int64_t)IB();
                    if (y == 0) { raise_exc(t, TPLX_EC_ZERODIVISIONERROR, opidx); break; }
                    R(rb, dst) = (uint64_t)floordiv_i64((int64_t)IA(), y);
                    break;
                }
                case TPLX_OP_IMOD: {
                    int64_t y = (int64_t)IB();
                    if (y == 0) { raise_exc(t, TPLX_EC_ZERODIVISIONERROR, opidx); break; }
                    R(rb, dst) = (uint64_t)floormod_i64((int64_t)IA(), y);
                    break;
                }
                case TPLX_OP_INEG: R(rb, dst) = (uint64_t)0 - IA(); break;
                case TPLX_OP_IAND: R(rb, dst) = IA() & IB(); break;
                case TPLX_OP_IOR: R(rb, dst) = IA() | IB(); break;
                case TPLX_OP_IXOR: R(rb, dst) = IA() ^ IB(); break;
                case TPLX_OP_ISHL: R(rb, dst) = IA() << (IB() & 63); break;
                case TPLX_OP_ISHR: R(rb, dst) = (uint64_t)((int64_t)IA() >> (IB() & 63)); break;
                case TPLX_OP_IABS: {
                    int64_t x = (int64_t)IA();
                    R(rb, dst) = (uint64_t)(x < 0 ? (uint64_t)0 - (uint64_t)x : (uint64_t)x);
                    break;
                }
                // single-rounded IEEE ops; the _rn intrinsics are never contracted into FMA
                case TPLX_OP_FADD: WF(__dadd_rn(FA(), FB())); break;
                case TPLX_OP_FSUB: WF(__dsub_rn(FA(), FB())); break;
                case TPLX_OP_FMUL: WF(__dmul_rn(FA(), FB())); break;
                case TPLX_OP_FDIV: {
                    double y = FB();
                    if (y == 0.0) { raise_exc(t, TPLX_EC_ZERODIVISIONERROR, opidx); break; }
                    WF(__ddiv_rn(FA(), y));
                    break;
                }
                case TPLX_OP_FMOD: {
                    double x = FA(), y = FB();
                    if (y == 0.0) { raise_exc(t, TPLX_EC_ZERODIVISIONERROR, opidx); break; }
                    WF(op_fmod(x, y));
                    break;
                }
                case TPLX_OP_FNEG: R(rb, dst) = IA() ^ 0x8000000000000000ull; break;
                case TPLX_OP_FABS: R(rb, dst) = IA() & 0x7FFFFFFFFFFFFFFFull; break;
                case TPLX_OP_FFLOORDIV: {
                    double y = FB();
                    if (y == 0.0) { raise_exc(t, TPLX_EC_ZERODIVISIONERROR, opidx); break; }
                    int64_t xi = (int64_t)FA(), yi = (int64_t)y;
                    if (yi == 0) { raise_exc(t, TPLX_EC_ZERODIVISIONERROR, opidx); break; }
                    WF((double)floordiv_i64(xi, yi));
                    break;
                }
                case TPLX_OP_I2F: WF((double)(int64_t)IA()); break;
                case TPLX_OP_F2I: R(rb, dst) = (uint64_t)(int64_t)FA(); break;
                case TPLX_OP_ICMP: R(rb, dst) = op_icmp(flags & 7, (int64_t)IA(), (int64_t)IB()); break;
                case TPLX_OP_FCMP: R(rb, dst) = op_fcmp(flags & 7, FA(), FB()); break;
                case TPLX_OP_BAND: R(rb, dst) = (IA() != 0) & (IB() != 0); break;
                case TPLX_OP_BOR: R(rb, dst) = (IA() != 0) | (IB() != 0); break;
                case TPLX_OP_BNOT: R(rb, dst) = (IA() == 0); break;
                case TPLX_OP_SLEN: R(rb, dst) = (uint64_t)SA().len; break;
                case TPLX_OP_SFIND: R(rb, dst) = (uint64_t)str_find(SA(), SB()); break;
                case TPLX_OP_SRFIND: R(rb, dst) = (uint64_t)str_rfind(SA(), SB()); break;
                case TPLX_OP_SFINDE: {  // find, or len(a) when absent
                    const StrV s = SA();
                    const int64_t r = str_find(s, SB());
                    R(rb, dst) = r < 0 ? (uint64_t)s.len : (uint64_t)r;
                    break;
                }
                case TPLX_OP_SRFINDK: {  // rfind + K, or 0 when absent
                    const int64_t r = str_rfind(RS(rb, a), SB());
                    R(rb, dst) = r < 0 ? 0ull : (uint64_t)r + (uint64_t)prog[pc].imm2;
                    break;
                }
                case TPLX_OP_SIN: R(rb, dst) = str_find(SB(), SA()) >= 0; break;
                case TPLX_OP_SEQ: R(rb, dst) = (uint64_t)(str_eq(SA(), SB()) != (bool)(flags & 1)); break;
                case TPLX_OP_STRUTH: R(rb, dst) = SA().len != 0; break;
                case TPLX_OP_SSTARTS: R(rb, dst) = op_sstarts(SA(), SB()); break;
                case TPLX_OP_SENDS: R(rb, dst) = op_sends(SA(), SB()); break;
                case TPLX_OP_SSLICE: {
                    const StrV o = op_sslice(SA(), flags, (flags & TPLX_SL_HAS_START) ? (int64_t)IB() : 0, (flags & TPLX_SL_HAS_END) ? (int64_t)IC() : 0);
                    WS(rb, dst, o.p, o.len, o.flags);
                    break;
                }
                case TPLX_OP_SINDEX: {
                    StrV o;
                    if (!op_sindex(SA(), (int64_t)IB(), &o)) { raise_exc(t, TPLX_EC_INDEXERROR, opidx); break; }
                    WS(rb, dst, o.p, o.len, o.flags);
                    break;
                }
                case TPLX_OP_SLOWER: {
                    StrV s = SA();
                    WS(rb, dst, s.p, s.len, TPLX_SF_LOWER);
                    break;
                }
                case TPLX_OP_SUPPER: {
                    StrV s = SA();
                    WS(rb, dst, s.p, s.len, TPLX_SF_UPPER);
                    break;
                }
                case TPLX_OP_SSTRIP: {
                    const StrV o = op_sstrip(SA(), flags);
                    WS(rb, dst, o.p, o.len, o.flags);
                    break;
                }
                case TPLX_OP_SCONCAT: {
                    StrV o;
                    if (!op_sconcat(t, SA(), SB(), opidx, &o)) break;
                    WS(rb, dst, o.p, o.len, o.flags);
                    break;
                }
                case TPLX_OP_SREPLACE: {
                    StrV o;
                    if (!op_sreplace(t, SA(), SB(), SC(), opidx, &o)) break;
                    WS(rb, dst, o.p, o.len, o.flags);
                    break;
                }
                case TPLX_OP_SFMTD: {
                    StrV o;
                    if (!op_sfmtd(t, flags, R(rb, a), (uint32_t)imm, opidx, &o)) break;
                    WS(rb, dst, o.p, o.len, o.flags);
                    break;
                }
                case TPLX_OP_I2S: {
                    StrV o;
                    if (!op_i2s(t, (int64_t)R(rb, a), opidx, &o)) break;
                    WS(rb, dst, o.p, o.len, o.flags);
                    break;
                }
                case TPLX_OP_S2I: {
                    int64_t v;
                    if (!str_to_i64(SA(), &v)) { raise_exc(t, TPLX_EC_VALUEERROR, opidx); break; }
                    R(rb, dst) = (uint64_t)v;
                    break;
                }
                case TPLX_OP_S2F: {
                    const StrV s = SA();
                    double d;
                    if (!str_to_f64(s, &d)) { raise_exc(t, TPLX_EC_VALUEERROR, opidx); break; }
                    WF(d);
                    break;
                }
                case TPLX_OP_FILTER:
                    if (R(rb, a) == 0) t.alive = false;
                    break;
                case TPLX_OP_RAISE: raise_exc(t, (uint32_t)imm, opidx); break;
                default: break;
            }
#undef IA
#undef IB
#undef IC
#undef FA
#undef FB
#undef SA
#undef SB
#undef SC
#undef WF
        }
    }
};

}  // namespace tplx
