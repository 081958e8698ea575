// mask.cuh — K1m: the selective head of a pipeline (the prefilter stage) as a pure map: one keep bit and one
// exception bit per input row, no scan, no staging of outputs, no block-wide barrier in the steady state.
//
// Replaces, for the rows a selective filter throws away, the JIT'd block loop + processRow of the reference
// (tuplex/core/src/physical/TuplexSourceTaskBuilder.cc:104-215, PipelineBuilder.cc:565-700): the reference evaluates
// the operators in order and leaves the row at the first false filter (filterOperation :615-700, `nRows = 0`);
// here the leading operators up to the selective filter run over every row and only the survivors reach the dense
// launch (kernels.cuh) that evaluates the whole stage and writes rows.
//
// Execution model: every WARP is autonomous. It owns warp-tiles of 32 consecutive rows (tile t -> warp t mod #warps),
// one row per lane, and reads the input columns from global memory: coalesced offsets, string bytes through L1. The kernel
// is issue-bound rather than latency-bound, so it spends no instructions on staging tiles in shared memory. The one
// block-wide barrier publishes the program and the column table.
// Results: keep_words[t] / exc_words[t] = warp ballots (bit l = row 32 t + l); exc_codes[row] for exception rows only.
// mask_count / mask_scan / mask_expand turn the bitmaps into the ascending survivor list and the exception records.
#pragma once
#include <stdint.h>
#include "kernels.cuh"

namespace tplx {

constexpr uint32_t MASK_WARPS = NT / 32;

struct MaskParams {
    uint64_t n_rows;
    uint32_t n_instr, n_in, n_slots, n_tiles;  // n_tiles = warp-tiles of 32 rows
    uint32_t scratch_per_thread;
    uint32_t smem_regs_off, smem_cols_off;
    const DInstr *prog;
    const uint8_t *cpool;
    uint32_t n_terms;                      // > 0: closed-form evaluation of the stage (string-scan hint), the program is not interpreted
    tplx_scan_term terms[TPLX_MAX_SCAN_TERMS];
    uint32_t *keep_words, *exc_words;      // n_rows / 32 (rounded up) words each
    uint32_t *exc_codes;                   // n_rows entries, written for exception rows only: code | opidx << 16
    uint8_t *scratch;
    ColIn in[TPLX_MAX_COLS];
};

// ---- K1f: closed-form evaluation of a string-scan hint (include/tplx_ir.h tplx_scan_term) ---------------------------------------
// The same string primitives as the VM's ops (strops.cuh), called directly: no instruction fetch / decode / register file.
template <uint32_t HF>
__device__ __forceinline__ int64_t scan_find(const StrV &h, const StrV &n) {
    if (n.len == 0) return 0;
    if (n.len > h.len) return -1;
    return str_find_impl<HF>(h, n);
}
__device__ __forceinline__ bool cmp_i64(uint32_t cmp, int64_t x, int64_t y) {
    switch (cmp) {
        case TPLX_CMP_EQ: return x == y;
        case TPLX_CMP_NE: return x != y;
        case TPLX_CMP_LT: return x < y;
        case TPLX_CMP_LE: return x <= y;
        case TPLX_CMP_GT: return x > y;
        default: return x >= y;
    }
}
__device__ __forceinline__ bool cmp_f64(uint32_t cmp, double x, double y) {  // ordered predicates (FCMP_O*), != is FCMP_ONE
    switch (cmp) {
        case TPLX_CMP_EQ: return x == y;
        case TPLX_CMP_NE: return (x < y) || (x > y);
        case TPLX_CMP_LT: return x < y;
        case TPLX_CMP_LE: return x <= y;
        case TPLX_CMP_GT: return x > y;
        default: return x >= y;
    }
}
__device__ __forceinline__ StrV scan_col(const ColIn &ci, uint64_t row) {
    StrV s;
    // the column lives in global memory, so the string primitives can use LDG instead of generic LD
    __builtin_assume(__isGlobal(ci.data));
    __builtin_assume(__isGlobal(ci.offsets));
    const uint32_t o0 = ci.offsets[row], o1 = ci.offsets[row + 1];
    s.p = reinterpret_cast<const uint8_t *>(ci.data) + o0;
    s.len = o1 - o0;
    s.flags = 0;
    return s;
}
__device__ __forceinline__ StrV scan_const(const uint8_t *cpool, uint64_t enc) {
    StrV v;
    v.p = cpool + (uint32_t)enc;
    v.len = (uint32_t)(enc >> 32);
    v.flags = 0;
    return v;
}
// evaluates the terms in order for one row; a row raises only in a term it reaches (PipelineBuilder.cc:949)
__device__ __forceinline__ void scan_eval(const MaskParams &P, const ColIn *__restrict__ cols, uint64_t row, VMThread &t) {
    for (uint32_t k = 0; k < P.n_terms; ++k) {
        if (!__any_sync(0xFFFFFFFFu, t.alive)) break;
        const tplx_scan_term &T = P.terms[k];
        if (!t.alive) continue;
        const ColIn &ci = cols[T.col];
        if (T.kind == TPLX_SK_CONTAINS) {
            StrV s = scan_col(ci, row);
            const StrV n = scan_const(P.cpool, T.needle);
            const uint32_t cf = T.flags & TPLX_SCF_CASE_MASK;
            s.flags = cf;
            const int64_t r = cf == TPLX_SF_LOWER ? scan_find<TPLX_SF_LOWER>(s, n) : (cf == TPLX_SF_UPPER ? scan_find<TPLX_SF_UPPER>(s, n) : scan_find<TPLX_SF_NONE>(s, n));
            t.alive = (r >= 0) != ((T.flags & TPLX_SCF_NEGATE) != 0);
        } else if (T.kind == TPLX_SK_FIELD_INT) {
            const StrV s = scan_col(ci, row);
            const int64_t i = scan_find<TPLX_SF_NONE>(s, scan_const(P.cpool, T.needle));
            StrV head = s;
            head.len = i < 0 ? s.len : (uint32_t)i;                                   // s[:stop]
            const StrV sep = scan_const(P.cpool, T.sep);
            int64_t j = -1;
            if (sep.len <= head.len) j = sep.len == 0 ? (int64_t)head.len : str_rfind_impl<TPLX_SF_NONE>(head, sep);
            const int64_t st = slice_index(j < 0 ? 0 : j + T.skip, (int64_t)head.len);  // head[start:] with Python's clamping
            StrV f;
            f.p = head.p + st;
            f.len = (uint32_t)((int64_t)head.len - st);
            f.flags = 0;
            int64_t v;
            if (!str_to_i64(f, &v)) {
                t.exc_code = TPLX_EC_VALUEERROR;
                t.exc_op = T.opidx_val;
                t.alive = false;
            } else t.alive = cmp_i64(T.cmp, v, T.imm);
        } else {
            const uint64_t raw = reinterpret_cast<const uint64_t *>(ci.data)[row];
            t.alive = (T.flags & TPLX_SCF_F64) ? cmp_f64(T.cmp, __longlong_as_double((long long)raw), __longlong_as_double((long long)T.imm))
                                               : cmp_i64(T.cmp, (int64_t)raw, T.imm);
        }
    }
}

// The parameter block travels by value in the kernel's constant bank (__grid_constant__): every P.field below is a constant-bank
// operand instead of a global load through a pointer (terms, column table, offsets — read in the per-row loops).
// __launch_bounds__(NT, 4): 4 resident CTAs per SM, 64 registers per thread.
#if !defined(TPLX_JIT) || TPLX_JIT_KIND == 5
#ifdef TPLX_JIT
// specialised K1m (stage specialiser, jit.inl): the prefilter program as straight-line code, no register file at all (the bitmaps carry the result)
extern "C" __global__ void __launch_bounds__(NT, TPLX_JIT_MIN_CTAS) tplx_jit_kernel(const __grid_constant__ MaskParams P) {
    constexpr bool SCAN = false;
#else
template <bool SCAN>
__global__ void __launch_bounds__(NT, 4) stage_mask_kernel(const __grid_constant__ MaskParams P) {
#endif
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    DInstr *s_prog = reinterpret_cast<DInstr *>(smem);
    uint8_t *s_regs = smem + P.smem_regs_off + tid * 8;
    ColIn *s_cols = reinterpret_cast<ColIn *>(smem + P.smem_cols_off);

    if (!SCAN)
        for (uint32_t i = tid; i < P.n_instr * (sizeof(DInstr) / 16); i += NT)
            reinterpret_cast<uint4 *>(s_prog)[i] = reinterpret_cast<const uint4 *>(P.prog)[i];
    for (uint32_t i = tid; i < P.n_in * (sizeof(ColIn) / 8); i += NT)
        reinterpret_cast<uint64_t *>(s_cols)[i] = reinterpret_cast<const uint64_t *>(P.in)[i];
    __syncthreads();  // the only block-wide barrier: program + column table ready

    VMThread t;
    t.scr_cap = P.scratch_per_thread;
    t.scratch = P.scratch + ((size_t)blockIdx.x * NT + tid) * (size_t)P.scratch_per_thread;

    const uint32_t gw = blockIdx.x * MASK_WARPS + warp, GW = gridDim.x * MASK_WARPS;
    const uint32_t my_tiles = P.n_tiles > gw ? (P.n_tiles - gw + GW - 1) / GW : 0;
    for (uint32_t q = 0; q < my_tiles; ++q) {
        const uint64_t tile = gw + (uint64_t)q * GW;
        const uint64_t row = tile * 32 + lane;
        t.alive = row < P.n_rows;
        t.exc_code = 0;
        t.scr_used = 0;
        if (SCAN) scan_eval(P, s_cols, row, t);
        else TPLX_VM_RUN(s_prog, P.n_instr, s_regs, s_cols, row, row, P.cpool, t);
        const bool exc = t.exc_code != 0;
        const uint32_t kb = __ballot_sync(0xFFFFFFFFu, t.alive);
        const uint32_t eb = __ballot_sync(0xFFFFFFFFu, exc);
        if (lane == 0) {
            P.keep_words[tile] = kb;
            P.exc_words[tile] = eb;
        }
        if (exc) P.exc_codes[row] = t.exc_code | (t.exc_op << 16);
    }
}
#endif  // K1m

#ifndef TPLX_JIT

// ---------------------------------------------------------------------------------------------------------
// bitmaps -> ascending survivor list + exception records (three small launches; the bitmaps are n_rows / 8 bytes)
// ---------------------------------------------------------------------------------------------------------
constexpr uint32_t CMP_NT = 1024;

__device__ __forceinline__ uint2 block_scan_pair(uint32_t a, uint32_t b, uint32_t *s_w /* 2 * 32 */, uint2 &total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, ia, o), y = __shfl_up_sync(0xFFFFFFFFu, ib, o);
        if (lane >= (uint32_t)o) { ia += x; ib += y; }
    }
    if (lane == 31) { s_w[warp] = ia; s_w[32 + warp] = ib; }
    __syncthreads();
    if (warp == 0) {
        uint32_t wa = s_w[lane], wb = s_w[32 + lane], ja = wa, jb = wb;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, ja, o), y = __shfl_up_sync(0xFFFFFFFFu, jb, o);
            if (lane >= (uint32_t)o) { ja += x; jb += y; }
        }
        s_w[lane] = ja - wa;
        s_w[32 + lane] = jb - wb;
        if (lane == 31) { s_w[64] = ja; s_w[65] = jb; }
    }
    __syncthreads();
    total = make_uint2(s_w[64], s_w[65]);
    return make_uint2(s_w[warp] + ia - a, s_w[32 + warp] + ib - b);  // exclusive prefixes inside the block
}

__global__ void __launch_bounds__(CMP_NT) mask_count_kernel(const uint32_t *__restrict__ keep, const uint32_t *__restrict__ exc, uint32_t n_words,
                                                            uint64_t *__restrict__ part) {
    __shared__ uint32_t s_w[66];
    const uint32_t w = blockIdx.x * CMP_NT + threadIdx.x;
    const uint32_t a = w < n_words ? __popc(keep[w]) : 0, b = w < n_words ? __popc(exc[w]) : 0;
    uint2 tot;
    block_scan_pair(a, b, s_w, tot);
    if (threadIdx.x == 0) { part[2 * blockIdx.x] = tot.x; part[2 * blockIdx.x + 1] = tot.y; }
}

// one CTA: exclusive scan of the per-block totals in place, grand totals -> totals[0..1]
__global__ void __launch_bounds__(CMP_NT) mask_scan_kernel(uint64_t *__restrict__ part, uint32_t nb, uint64_t *__restrict__ totals) {
    __shared__ uint32_t s_w[66];
    uint64_t ca = 0, cb = 0;
    for (uint32_t base = 0; base < nb; base += CMP_NT) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t a = i < nb ? (uint32_t)part[2 * i] : 0, b = i < nb ? (uint32_t)part[2 * i + 1] : 0;
        uint2 tot;
        const uint2 ex = block_scan_pair(a, b, s_w, tot);
        if (i < nb) { part[2 * i] = ca + ex.x; part[2 * i + 1] = cb + ex.y; }
        ca += tot.x;
        cb += tot.y;
        __syncthreads();
    }
    if (threadIdx.x == 0) { totals[0] = ca; totals[1] = cb; }
}

__global__ void __launch_bounds__(CMP_NT) mask_expand_kernel(const uint32_t *__restrict__ keep, const uint32_t *__restrict__ exc, uint32_t n_words,
                                                             const uint64_t *__restrict__ part, uint64_t *__restrict__ rowlist,
                                                             const uint32_t *__restrict__ exc_codes, const int64_t *__restrict__ opids,
                                                             tplx_exception_rec *__restrict__ exc_out, uint64_t cap_exc) {
    __shared__ uint32_t s_w[66];
    const uint32_t w = blockIdx.x * CMP_NT + threadIdx.x;
    uint32_t kw = w < n_words ? keep[w] : 0, ew = w < n_words ? exc[w] : 0;
    uint2 tot;
    const uint2 ex = block_scan_pair(__popc(kw), __popc(ew), s_w, tot);
    uint64_t ko = part[2 * blockIdx.x] + ex.x, eo = part[2 * blockIdx.x + 1] + ex.y;
    while (kw) {
        const uint32_t bit = __ffs(kw) - 1;
        kw &= kw - 1;
        rowlist[ko++] = (uint64_t)w * 32 + bit;
    }
    while (ew) {
        const uint32_t bit = __ffs(ew) - 1;
        ew &= ew - 1;
        const uint64_t row = (uint64_t)w * 32 + bit;
        const uint32_t es = exc_codes[row];
        tplx_exception_rec rec;
        rec.row = (int64_t)row;
        rec.row_no = 0;  // numbered by the caller once the dense launch's rows are known
        rec.code = es & 0xFFFF;
        rec.op_id = opids[es >> 16];
        if (eo < cap_exc) exc_out[eo] = rec;  // beyond the estimated capacity: the host sees totals[1] > cap and expands again
        ++eo;
    }
}

#endif  // !TPLX_JIT

}  // namespace tplx
