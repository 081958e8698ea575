// mask.cuh — K1m: the selective head of a pipeline (the prefilter stage) as a pure map: one keep bit and one
// exception bit per input row, no scan, no staging of outputs, no block-wide barrier in the steady state.
//
// Replaces, for the rows a selective filter throws away, the JIT'd block loop + processRow of the reference
// (tuplex/core/src/physical/TuplexSourceTaskBuilder.cc:104-215, PipelineBuilder.cc:565-700): the reference evaluates
// the operators in order and leaves the row at the first false filter (filterOperation :615-700, `nRows = 0`);
// here the leading operators up to the selective filter run over every row and only the survivors reach the dense
// launch (kernels.cuh) that evaluates the whole stage and writes rows.
//
// Execution model: every WARP is autonomous. It owns warp-tiles of 32*MR consecutive rows (tile t -> warp
// t mod #warps), a private 2-deep shared-memory ring, and one mbarrier per ring slot. For tile k+1 the lanes
// 0..n_staged-1 each bring one string column's byte range [offsets[r0], offsets[r1]) and its offsets into the ring
// with cp.async.bulk (TMA bulk copy, SASS UBLKCP; completion counted on the mbarrier), while the warp evaluates
// tile k out of shared memory: the VM's string primitives then read shared memory (~30 cycles) instead of
// L2/HBM. A tile whose byte range exceeds the ring slot simply keeps its global pointers (always correct).
// Results: keep_words[t] / exc_words[t] = warp ballots (bit l = row 32 t + l); exc_codes[row] for exception rows only.
// mask_count / mask_scan / mask_expand turn the bitmaps into the ascending survivor list and the exception records.
#pragma once
#include <stdint.h>
#include "kernels.cuh"
#include "fused.cuh"

namespace tplx {

constexpr uint32_t MASK_MAX_STAGED = 4;
constexpr uint32_t MASK_WARPS = NT / 32;
constexpr uint32_t MASK_RING = 2;

struct MaskParams {
    uint64_t n_rows;
    uint32_t n_instr, n_in, n_slots, n_tiles;  // n_tiles = warp-tiles of 32*MR rows
    uint32_t n_staged, MR;
    uint32_t scratch_per_thread;
    uint32_t smem_regs_off, smem_wcols_off, smem_bar_off, smem_info_off, smem_ring_off;
    uint32_t slot_bytes;                   // one ring slot of one warp (all staged columns)
    uint32_t off_bytes;                    // bytes of the staged offsets of one column: (32*MR + 1) * 4 rounded up to 16
    uint32_t st_col[MASK_MAX_STAGED];      // input column of each staged column
    uint32_t st_cap[MASK_MAX_STAGED];      // byte capacity (multiple of 16) of its string bytes in a ring slot
    uint32_t st_boff[MASK_MAX_STAGED];     // where its bytes live inside a ring slot
    uint32_t st_ooff[MASK_MAX_STAGED];     // where its offsets live inside a ring slot
    const DInstr *prog;
    const uint8_t *cpool;
    uint32_t n_terms;                      // > 0: closed-form evaluation of the stage (string-scan hint), the program is not interpreted
    tplx_scan_term terms[TPLX_MAX_SCAN_TERMS];
    uint32_t *keep_words, *exc_words;      // n_rows / 32 (rounded up) words each
    uint32_t *exc_codes;                   // n_rows entries, written for exception rows only: code | opidx << 16
    uint8_t *scratch;
    ColIn in[TPLX_MAX_COLS];
};

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

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
template <bool GLOBAL_ONLY>
__device__ __forceinline__ StrV scan_col(const ColIn &ci, uint64_t row) {
    StrV s;
    if (GLOBAL_ONLY) {  // nothing is staged: the column lives in global memory, so the string primitives can use LDG instead of generic LD
        __builtin_assume(__isGlobal(ci.data));
        __builtin_assume(__isGlobal(ci.offsets));
    }
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
template <bool GLOBAL_ONLY>
__device__ __forceinline__ void scan_eval(const MaskParams &P, const ColIn *__restrict__ cols, uint64_t row, VMThread &t) {
    for (uint32_t k = 0; k < P.n_terms; ++k) {
        if (!__any_sync(0xFFFFFFFFu, t.alive)) break;
        const tplx_scan_term &T = P.terms[k];
        if (!t.alive) continue;
        const ColIn &ci = cols[T.col];
        if (T.kind == TPLX_SK_CONTAINS) {
            StrV s = scan_col<GLOBAL_ONLY>(ci, row);
            const StrV n = scan_const(P.cpool, T.needle);
            const uint32_t cf = T.flags & TPLX_SCF_CASE_MASK;
            s.flags = cf;
            const int64_t r = cf == TPLX_SF_LOWER ? scan_find<TPLX_SF_LOWER>(s, n) : (cf == TPLX_SF_UPPER ? scan_find<TPLX_SF_UPPER>(s, n) : scan_find<TPLX_SF_NONE>(s, n));
            t.alive = (r >= 0) != ((T.flags & TPLX_SCF_NEGATE) != 0);
        } else if (T.kind == TPLX_SK_FIELD_INT) {
            const StrV s = scan_col<GLOBAL_ONLY>(ci, row);
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
// MINB: resident CTAs per SM the register allocation must allow (4 = 64 registers, 5 = 48, 6 = 40).
#if !defined(TPLX_JIT) || TPLX_JIT_KIND == 5
#ifdef TPLX_JIT
// specialised K1m (stage specialiser, jit.inl): the prefilter program as straight-line code, no register file at all (the bitmaps carry the result)
extern "C" __global__ void __launch_bounds__(NT, TPLX_JIT_MINB) tplx_jit_kernel(const __grid_constant__ MaskParams P) {
    constexpr bool SCAN = false;
#else
template <bool SCAN, int MINB = 4>
__global__ void __launch_bounds__(NT, MINB) stage_mask_kernel(const __grid_constant__ MaskParams P) {
#endif
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t MR = P.MR, TR = 32 * MR, ns = P.n_staged;

    DInstr *s_prog = reinterpret_cast<DInstr *>(smem);
    uint8_t *s_regs = smem + P.smem_regs_off + tid * 8;
    ColIn *s_wcols = reinterpret_cast<ColIn *>(smem + P.smem_wcols_off) + warp * P.n_in;          // this warp's column table
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + P.smem_bar_off) + warp * MASK_RING;
    uint32_t *info = reinterpret_cast<uint32_t *>(smem + P.smem_info_off) + warp * MASK_RING * 2 * MASK_MAX_STAGED;
    uint8_t *ring = smem + P.smem_ring_off + (size_t)warp * MASK_RING * P.slot_bytes;

    if (!SCAN)
        for (uint32_t i = tid; i < P.n_instr * (sizeof(DInstr) / 16); i += NT)
            reinterpret_cast<uint4 *>(s_prog)[i] = reinterpret_cast<const uint4 *>(P.prog)[i];
    for (uint32_t i = lane; i < P.n_in * (sizeof(ColIn) / 8); i += 32)
        reinterpret_cast<uint64_t *>(s_wcols)[i] = reinterpret_cast<const uint64_t *>(P.in)[i];
    if (lane == 0 && ns) {
        for (uint32_t s = 0; s < MASK_RING; ++s) mbar_init(&bars[s], ns);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();  // the only block-wide barrier: program + barriers ready

    VMThread t;
    t.scr_cap = P.scratch_per_thread;
    t.scratch = P.scratch + ((size_t)blockIdx.x * NT + tid) * (size_t)P.scratch_per_thread;

    const uint32_t gw = blockIdx.x * MASK_WARPS + warp, GW = gridDim.x * MASK_WARPS;
    const uint32_t my_tiles = P.n_tiles > gw ? (P.n_tiles - gw + GW - 1) / GW : 0;

    // lane k < ns stages column st_col[k] of a tile into ring slot `slot`
    const bool stager = lane < ns;
    const ColIn my_col = stager ? P.in[P.st_col[lane]] : ColIn{};
    const bool offs_aligned = stager && ((reinterpret_cast<uintptr_t>(my_col.offsets) & 15) == 0);
    auto issue = [&](uint32_t q, uint32_t o0, uint32_t o1) {
        const uint32_t slot = q % MASK_RING;
        const uint64_t r0 = (uint64_t)(gw + (uint64_t)q * GW) * TR;
        const uint32_t a0 = o0 & ~15u;
        const uint32_t nb = ((o1 + 15u) & ~15u) - a0;
        const bool sb = nb != 0 && nb <= P.st_cap[lane];
        const bool so = offs_aligned && r0 + P.off_bytes / 4 <= P.n_rows + 1;
        uint32_t *inf = info + slot * 2 * MASK_MAX_STAGED;
        inf[lane] = sb ? a0 : 0xFFFFFFFFu;
        inf[MASK_MAX_STAGED + lane] = so;
        mbar_arrive_expect_tx(&bars[slot], (sb ? nb : 0u) + (so ? P.off_bytes : 0u));
        uint8_t *dst = ring + (size_t)slot * P.slot_bytes;
        if (sb) bulk_g2s(dst + P.st_boff[lane], reinterpret_cast<const uint8_t *>(my_col.data) + a0, nb, &bars[slot]);
        if (so) bulk_g2s(dst + P.st_ooff[lane], my_col.offsets + r0, P.off_bytes, &bars[slot]);
    };
    auto tile_range = [&](uint32_t q, uint32_t &o0, uint32_t &o1) {  // byte range of tile q of this warp in my column
        const uint64_t r0 = (uint64_t)(gw + (uint64_t)q * GW) * TR;
        const uint64_t r1 = r0 + TR < P.n_rows ? r0 + TR : P.n_rows;
        o0 = my_col.offsets[r0];
        o1 = my_col.offsets[r1];
    };
    uint32_t no0 = 0, no1 = 0;  // range of the next tile to issue (loaded one iteration ahead)
    if (stager && my_tiles) {
        tile_range(0, no0, no1);
        issue(0, no0, no1);
        if (my_tiles > 1) tile_range(1, no0, no1);
    }

    for (uint32_t q = 0; q < my_tiles; ++q) {
        const uint32_t slot = q % MASK_RING;
        const uint64_t tile = gw + (uint64_t)q * GW;
        const uint64_t r0 = tile * TR;
        if (ns) {
            if (stager && q + 1 < my_tiles) {
                issue(q + 1, no0, no1);  // slot (q+1)%2 was released by the __syncwarp that ended iteration q-1
                if (q + 2 < my_tiles) tile_range(q + 2, no0, no1);
            }
            mbar_wait(&bars[slot], (q / MASK_RING) & 1);
            if (stager) {
                const uint32_t *inf = info + slot * 2 * MASK_MAX_STAGED;
                const uint32_t a0 = inf[lane];
                const uint8_t *base = ring + (size_t)slot * P.slot_bytes;
                ColIn &wc = s_wcols[P.st_col[lane]];
                // views are formed as data + offsets[row]: rebase both so that the sums land inside the ring slot
                wc.data = a0 != 0xFFFFFFFFu ? static_cast<const void *>(base + P.st_boff[lane] - a0) : my_col.data;
                wc.offsets = inf[MASK_MAX_STAGED + lane] ? reinterpret_cast<const uint32_t *>(base + P.st_ooff[lane]) - r0 : my_col.offsets;
            }
            __syncwarp();
        }
        for (uint32_t s = 0; s < MR; ++s) {
            const uint64_t row = r0 + (uint64_t)s * 32 + lane;
            t.alive = row < P.n_rows;
            t.exc_code = 0;
            t.scr_used = 0;
            if (SCAN) { if (ns) scan_eval<false>(P, s_wcols, row, t); else scan_eval<true>(P, s_wcols, row, t); }
            else TPLX_VM_RUN(s_prog, P.n_instr, s_regs, s_wcols, row, row, P.cpool, t);
            const bool exc = t.exc_code != 0;
            const uint32_t kb = __ballot_sync(0xFFFFFFFFu, t.alive);
            const uint32_t eb = __ballot_sync(0xFFFFFFFFu, exc);
            if (lane == 0) {
                P.keep_words[tile * MR + s] = kb;
                P.exc_words[tile * MR + s] = eb;
            }
            if (exc) P.exc_codes[row] = t.exc_code | (t.exc_op << 16);
        }
        __syncwarp();  // every lane is done with this ring slot
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
