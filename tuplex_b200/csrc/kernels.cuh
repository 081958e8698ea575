// kernels.cuh — stage kernels for sm_90a.
//
// K1  stage_rows_kernel   : fused map/filter/withColumn/project over a column block, stable
//                           compaction (warp ballot bitmaps) + single-pass decoupled look-back scan
//                           for output row / string byte / exception offsets. Replaces the JIT'd
//                           block loop + processRow + writeRowToMemory
//                           (reference tuplex/core/src/physical/TuplexSourceTaskBuilder.cc:104-215,
//                            PipelineBuilder.cc:565-1025, core/include/physical/TransformTask.h:47-92).
// K2  exception records are emitted by K1 itself (row, rowNo, code, opID); the original row bytes are
//     gathered by rowfmt.cuh (IExceptionableTask.h:22-36).
// K3  stage_agg_kernel + agg_finalize_kernel : fused filter -> g(x) -> fixed-tree reduction.
//     Replaces addAggregate/combineAggregate/fetchAggregate
//     (PipelineBuilder.cc:2525-2608, TransformTask.cc:218-299).
#pragma once
#include <stdint.h>
#include "vm.cuh"
#include "../../include/tplx_gpu.h"

namespace tplx {

constexpr int NT = 256;           // threads per CTA
constexpr int MAX_SCAN = 32;      // look-back vector width: keep, exc, + string output columns
constexpr int FIN_NT = 1024;      // finalize CTA width

struct OutCol {
    uint64_t *data;      // fixed-width values
    uint32_t *offsets;   // string: n_out+1 offsets
    uint8_t *bytes;      // string bytes
    uint64_t cap_bytes;  // capacity of bytes
    uint32_t slot;
    uint32_t type;
    int32_t strk;        // index among string output columns, -1 for fixed width
    uint32_t stage_off;  // byte offset of this column's staging area in shared memory
};

struct AccP {
    uint32_t kind;
    uint32_t slot;
    int64_t init;
};

struct KParams {
    uint64_t n_rows;
    int64_t first_row_no;
    uint32_t n_instr;
    uint32_t inplace;         // 1: one row per thread and no staging area — outputs are read from the register file (slot s of local row lr = regs[s][lr])
    uint32_t n_slots, n_in, n_out, n_str_out, n_accs, R, n_tiles, scratch_per_thread;
    uint32_t K;            // scan vector width = 2 + n_str_out
    uint32_t smem_regs_off, smem_stage_off, smem_misc_off, smem_cols_off;
    uint32_t smem_stash_off;  // per string output column: NT/32 warp totals of the byte scan
    uint64_t cap_rows, cap_exc;
    const DInstr *prog;    // pre-decoded program (device format)
    const uint8_t *cpool;
    const int64_t *opids;
    uint64_t *tile_state;   // n_tiles * (1 + 2K)
    uint32_t *counters;     // [0] ticket, [1] overflow flags, [2] exception append counter (agg)
    uint64_t *totals;       // K totals
    tplx_exception_rec *exc;
    uint8_t *scratch;
    uint64_t *tile_partials;  // aggregate: n_tiles * n_accs
    uint64_t *agg_out;        // aggregate: n_accs
    const uint64_t *rowlist;  // optional: evaluate these input rows only (output of a prefilter stage), ascending
    uint64_t n_work;          // rows to evaluate: n_rows, or the length of rowlist (its CAPACITY when n_work_dev is set)
    const uint64_t *n_work_dev;  // optional: the actual length of rowlist lives on the device (written by an earlier kernel of the
                                 // same stream): the host sized everything from an estimate and never waited for the count
    ColIn in[TPLX_MAX_COLS];
    OutCol out[TPLX_MAX_COLS];
    AccP accs[TPLX_MAX_ACCS];
};

// ---- small helpers --------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t *p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_cg_u64(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_cg_u64(uint64_t *p, uint64_t v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

// accumulate one value into an accumulator (identity handling by kind)
__device__ __forceinline__ uint64_t acc_identity(uint32_t kind) {
    switch (kind) {
        case TPLX_ACC_SUM_I64: return 0;
        case TPLX_ACC_SUM_F64: return 0;  // +0.0
        case TPLX_ACC_MIN_I64: return 0x7FFFFFFFFFFFFFFFull;
        case TPLX_ACC_MAX_I64: return 0x8000000000000000ull;
        case TPLX_ACC_MIN_F64: return 0x7FF0000000000000ull;  // +inf
        default: return 0xFFF0000000000000ull;               // -inf
    }
}
__device__ __forceinline__ uint64_t acc_combine(uint32_t kind, uint64_t a, uint64_t b) {
    switch (kind) {
        case TPLX_ACC_SUM_I64: return a + b;
        case TPLX_ACC_SUM_F64:
            return (uint64_t)__double_as_longlong(
                __dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b)));
        case TPLX_ACC_MIN_I64: return (int64_t)b < (int64_t)a ? b : a;
        case TPLX_ACC_MAX_I64: return (int64_t)b > (int64_t)a ? b : a;
        case TPLX_ACC_MIN_F64:
            return __longlong_as_double((long long)b) < __longlong_as_double((long long)a) ? b : a;
        default: return __longlong_as_double((long long)b) > __longlong_as_double((long long)a) ? b : a;
    }
}

// rank of local row lr among set bits (exclusive)
__device__ __forceinline__ uint32_t bit_rank(const uint32_t *bits, const uint32_t *wpre, uint32_t lr) {
    return wpre[lr >> 5] + __popc(bits[lr >> 5] & ((1u << (lr & 31)) - 1u));
}
__device__ __forceinline__ bool bit_test(const uint32_t *bits, uint32_t lr) {
    return (bits[lr >> 5] >> (lr & 31)) & 1u;
}

// Tail of a tile, shared by the scalar (VM) and the vector (VecVM) row kernels: per-tile counts, decoupled look-back over the
// K-vector, stable compacted write of the staged outputs, exception records. On entry keep_bits / exc_bits / exc_stage and the
// staged output values (s_stage + out[c].stage_off, indexed by local row) are complete and a __syncthreads() has been passed.
struct TileSmem {
    uint8_t *s_stage, *s_regs;  // staging area (or the register file base when P.inplace), this thread's register column
    uint32_t *s_stash;          // [n_str_out][NT/32] warp totals of the string byte scan
    uint32_t *keep_bits, *exc_bits, *keep_pre, *exc_pre, *exc_stage;
    uint32_t exc_stride;        // exc_stage[lr * exc_stride]: 1, or 2 when the codes live in slot 0 of the raising row (in place)
    uint64_t *s_vals, *s_excl;
};
__device__ __forceinline__ void rows_tile_finish(const KParams &P, const TileSmem &S, uint32_t tile, uint64_t base, uint32_t R, uint32_t T,
                                                 uint32_t W, uint32_t K, uint32_t state_stride, uint32_t n_tiles) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint8_t *s_stage = S.s_stage;
    uint32_t *s_wtot = S.s_stash;
    // staged value of output column oc at local row lr: either the staging area ([lr] / [2 lr], [2 lr + 1]) or, in place, the register
    // file itself (slot-major: regs[slot][lr])
    auto fixed_at = [&](const OutCol &oc, uint32_t lr) -> uint64_t {
        return P.inplace ? reinterpret_cast<const uint64_t *>(s_stage + (size_t)oc.slot * (NT * 8))[lr]
                         : reinterpret_cast<const uint64_t *>(s_stage + oc.stage_off)[lr];
    };
    auto str_ptr_at = [&](const OutCol &oc, uint32_t lr) -> uint64_t {
        return P.inplace ? reinterpret_cast<const uint64_t *>(s_stage + (size_t)oc.slot * (NT * 8))[lr]
                         : reinterpret_cast<const uint64_t *>(s_stage + oc.stage_off)[2 * (size_t)lr];
    };
    auto str_meta_at = [&](const OutCol &oc, uint32_t lr) -> uint64_t {
        return P.inplace ? reinterpret_cast<const uint64_t *>(s_stage + (size_t)(oc.slot + 1) * (NT * 8))[lr]
                         : reinterpret_cast<const uint64_t *>(s_stage + oc.stage_off)[2 * (size_t)lr + 1];
    };
    uint32_t *keep_bits = S.keep_bits, *exc_bits = S.exc_bits, *keep_pre = S.keep_pre, *exc_pre = S.exc_pre, *exc_stage = S.exc_stage;
    uint64_t *s_vals = S.s_vals, *s_excl = S.s_excl;
    // ---- per-tile counts: word prefixes (warp 0), string byte totals ----------------------
    if (warp == 0) {
        uint32_t ck = 0, ce = 0;
        for (uint32_t w0 = 0; w0 < W; w0 += 32) {
            uint32_t w = w0 + lane;
            uint32_t pk = w < W ? __popc(keep_bits[w]) : 0, pe = w < W ? __popc(exc_bits[w]) : 0;
            uint32_t ik = pk, ie = pe;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t a = __shfl_up_sync(0xFFFFFFFFu, ik, o), b = __shfl_up_sync(0xFFFFFFFFu, ie, o);
                if (lane >= (uint32_t)o) { ik += a; ie += b; }
            }
            if (w < W) { keep_pre[w] = ck + ik - pk; exc_pre[w] = ce + ie - pe; }
            ck += __shfl_sync(0xFFFFFFFFu, ik, 31);
            ce += __shfl_sync(0xFFFFFFFFu, ie, 31);
        }
        if (lane == 0) {
            keep_pre[W] = ck;
            exc_pre[W] = ce;
            s_vals[0] = ck;
            s_vals[1] = ce;
        }
    }
    __syncthreads();
    const bool any_keep = s_vals[0] != 0;
    if (!any_keep && tid < MAX_SCAN - 2) s_vals[2 + tid] = 0;
    // string bytes per output column: thread owns local rows [tid*R, tid*R+R) (consecutive rows per thread, so that one block scan
    // yields in-order byte offsets). All columns are scanned between ONE pair of barriers; only the warp totals go through shared
    // memory — a thread's own exclusive offset is recomputed (one more warp scan) when the column is written.
    auto warp_scan_bytes = [&](const OutCol &oc, uint32_t &mine) -> uint32_t {  // inclusive scan of the thread's kept bytes over the warp
        mine = 0;
        for (uint32_t j = 0; j < R; ++j) {
            const uint32_t lr = tid * R + j;
            if (bit_test(keep_bits, lr)) mine += (uint32_t)str_meta_at(oc, lr);
        }
        uint32_t inc = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t a = __shfl_up_sync(0xFFFFFFFFu, inc, o);
            if (lane >= (uint32_t)o) inc += a;
        }
        return inc;
    };
    if (any_keep) {
        for (uint32_t c = 0; c < P.n_out; ++c) {
            const OutCol &oc = P.out[c];
            if (oc.strk < 0) continue;
            uint32_t mine;
            const uint32_t inc = warp_scan_bytes(oc, mine);
            if (lane == 31) s_wtot[(uint32_t)oc.strk * (NT / 32) + warp] = inc;
        }
        __syncthreads();
        if (tid < P.n_str_out) {
            uint32_t tot = 0;
            for (uint32_t w = 0; w < NT / 32; ++w) tot += s_wtot[tid * (NT / 32) + w];
            s_vals[2 + tid] = tot;
        }
    }
    __syncthreads();

    // ---- decoupled look-back over the K-vector (warp 0) -----------------------------------
    if (warp == 0) {
        uint64_t *my = P.tile_state + (size_t)tile * state_stride;
        uint64_t myval = lane < K ? s_vals[lane] : 0;
        if (lane < K) {
            st_cg_u64(my + 1 + lane, myval);
            if (tile == 0) st_cg_u64(my + 1 + K + lane, myval);
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) st_release_u32(reinterpret_cast<uint32_t *>(my), tile == 0 ? 2u : 1u);
        uint64_t excl = 0;
        if (tile > 0) {
            int64_t p = (int64_t)tile - 1;
            while (true) {
                const int64_t q = p - lane;
                uint32_t st = 2;
                const uint64_t *qs = nullptr;
                if (q >= 0) {
                    qs = P.tile_state + (size_t)q * state_stride;
                    do { st = ld_acquire_u32(reinterpret_cast<const uint32_t *>(qs)); } while (st == 0);
                }
                const uint32_t pm = __ballot_sync(0xFFFFFFFFu, st == 2);
                const uint32_t first = pm ? (uint32_t)(__ffs(pm) - 1) : 31u;
                const bool use = (lane <= first) && q >= 0;
                for (uint32_t k = 0; k < K; ++k) {
                    uint64_t v = use ? ld_cg_u64(qs + 1 + (st == 2 ? K : 0) + k) : 0;
                    v = warp_sum_u64(v);
                    if (lane == k) excl += v;
                }
                if (pm) break;
                p -= 32;
            }
            if (lane < K) st_cg_u64(my + 1 + K + lane, excl + myval);
            __threadfence();
            __syncwarp();
            if (lane == 0) st_release_u32(reinterpret_cast<uint32_t *>(my), 2u);
        }
        if (lane < K) {
            s_excl[lane] = excl;
            if (tile == n_tiles - 1) P.totals[lane] = excl + myval;
        }
    }
    __syncthreads();

    // ---- write ----------------------------------------------------------------------------
    const uint64_t pre_keep = s_excl[0], pre_exc = s_excl[1];
    const uint32_t n_keep = (uint32_t)s_vals[0], n_exc = (uint32_t)s_vals[1];
    const bool rows_fit = pre_keep + n_keep <= P.cap_rows;
    if (!rows_fit && tid == 0) atomicOr(&P.counters[1], 1u);
    if (n_keep && rows_fit) {
        for (uint32_t c = 0; c < P.n_out; ++c) {
            const OutCol &oc = P.out[c];
            if (oc.strk < 0) {
                for (uint32_t lr = tid; lr < T; lr += NT)
                    if (bit_test(keep_bits, lr)) oc.data[pre_keep + bit_rank(keep_bits, keep_pre, lr)] = fixed_at(oc, lr);
            } else {
                const uint64_t pre_b = s_excl[2 + oc.strk];
                const uint64_t tile_b = s_vals[2 + oc.strk];
                const bool fit = pre_b + tile_b <= oc.cap_bytes && pre_b + tile_b <= 0xFFFFFFFFull;
                if (!fit) {
                    if (tid == 0) atomicOr(&P.counters[1], 2u);
                    continue;
                }
                uint32_t mine, wofs = 0;
                const uint32_t inc = warp_scan_bytes(oc, mine);
                for (uint32_t w = 0; w < warp; ++w) wofs += s_wtot[(uint32_t)oc.strk * (NT / 32) + w];
                uint64_t off = pre_b + wofs + (inc - mine);  // this thread's exclusive byte offset
                for (uint32_t j = 0; j < R; ++j) {
                    const uint32_t lr = tid * R + j;
                    if (!bit_test(keep_bits, lr)) continue;
                    StrV sv;
                    sv.p = reinterpret_cast<const uint8_t *>(str_ptr_at(oc, lr));
                    const uint64_t m = str_meta_at(oc, lr);
                    sv.len = (uint32_t)m;
                    sv.flags = (uint32_t)(m >> 32);
                    oc.offsets[pre_keep + bit_rank(keep_bits, keep_pre, lr)] = (uint32_t)off;
                    str_copy(oc.bytes + off, sv);
                    off += sv.len;
                }
                if (tile == n_tiles - 1 && tid == 0) oc.offsets[pre_keep + n_keep] = (uint32_t)(pre_b + tile_b);
            }
        }
    } else if (tile == n_tiles - 1 && rows_fit && tid == 0) {
        for (uint32_t c = 0; c < P.n_out; ++c)
            if (P.out[c].strk >= 0) P.out[c].offsets[pre_keep] = (uint32_t)s_excl[2 + P.out[c].strk];
    }
    if (n_exc) {
        if (pre_exc + n_exc <= P.cap_exc) {
            for (uint32_t lr = tid; lr < T; lr += NT) {
                if (!bit_test(exc_bits, lr)) continue;
                const uint32_t ke = bit_rank(exc_bits, exc_pre, lr);
                const uint32_t kk = bit_rank(keep_bits, keep_pre, lr);
                tplx_exception_rec rec;
                rec.row = (int64_t)(P.rowlist ? P.rowlist[base + lr] : base + lr);
                // _outputRowCounter semantics: rows written + exceptions so far (TransformTask.cc:764,885)
                rec.row_no = P.first_row_no + (int64_t)(pre_keep + pre_exc + kk + ke);
                const uint32_t es = exc_stage[lr * S.exc_stride];
                rec.code = es & 0xFFFF;
                rec.op_id = P.opids[es >> 16];
                P.exc[pre_exc + ke] = rec;
            }
        } else if (tid == 0) atomicOr(&P.counters[1], 4u);
    }
}

// ---- stage specialiser (jit.inl) ----------------------------------------------------------------------------------------------
// When this header is compiled at run time by NVRTC (TPLX_JIT), "jit_row.cuh" is the op program of ONE stage printed as a
// straight-line function (jit_run / jit_row_fixed) and exactly one kernel of the library is compiled around it, as
// `tplx_jit_kernel`: TPLX_JIT_KIND 1 = K1 rows, 2 / 3 = K1v (J = 4 / 2), 4 = K3 aggregate, 5 = K1m mask, 6 = K1w, 10 = K1r
// (K4, the hash aggregate, is table-bound and stays interpreted). TPLX_JIT_MIN_CTAS is the kernel's second __launch_bounds__ argument.
// The register file of a specialised kernel is COMPACT: it holds the live-out slots only (outputs, accumulator inputs), in the
// order the host's jit::liveout() numbered them; KParams carries those compact slot numbers.
#ifdef TPLX_JIT
#include "jit_row.cuh"
#define TPLX_VM_RUN(prog, n_instr, regs, cols, row, w, cpool, t) jit_run(regs, cols, row, w, cpool, t)
#else
#define TPLX_VM_RUN(prog, n_instr, regs, cols, row, w, cpool, t) VM<NT>::run(prog, 0, n_instr, regs, cols, row, w, cpool, t)
#endif

// =============================================================================================
// K1: rows in -> rows out
// =============================================================================================
// Shared memory map (byte offsets from KParams): prog | cols | regs | staging | misc
// misc: keep_bits[W] exc_bits[W] keep_pre[W+1] exc_pre[W+1] exc_stage[T] scan scratch
#if !defined(TPLX_JIT) || TPLX_JIT_KIND == 1
#ifdef TPLX_JIT
extern "C" __global__ void __launch_bounds__(NT, TPLX_JIT_MIN_CTAS) tplx_jit_kernel(const __grid_constant__ KParams P) {
#else
__global__ void __launch_bounds__(NT) stage_rows_kernel(const __grid_constant__ KParams P) {  // parameters in the constant bank
#endif
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t R = P.R, T = R * NT, W = T / 32, K = P.K;

    DInstr *s_prog = reinterpret_cast<DInstr *>(smem);
    ColIn *s_cols = reinterpret_cast<ColIn *>(smem + P.smem_cols_off);
    uint8_t *s_regs = smem + P.smem_regs_off + tid * 8;  // this thread's register column
    uint8_t *s_stage = P.inplace ? smem + P.smem_regs_off : smem + P.smem_stage_off;
    uint32_t *s_stash = reinterpret_cast<uint32_t *>(smem + P.smem_stash_off);
    uint32_t *keep_bits = reinterpret_cast<uint32_t *>(smem + P.smem_misc_off);
    uint32_t *exc_bits = keep_bits + W;
    uint32_t *keep_pre = exc_bits + W;
    uint32_t *exc_pre = keep_pre + W + 1;
    // code | operator of a raising row: its own array, or (in place) slot 0 of that row in the register file — the row is not kept,
    // nobody reads its values any more
    uint32_t *exc_stage = P.inplace ? reinterpret_cast<uint32_t *>(smem + P.smem_regs_off) : exc_pre + W + 1;
    const uint32_t exc_stride = P.inplace ? 2u : 1u;
    uint64_t *s_vals = reinterpret_cast<uint64_t *>(exc_pre + W + 1 + (P.inplace ? 0u : T));  // K tile values
    uint64_t *s_excl = s_vals + MAX_SCAN;                                                    // K exclusive prefixes
    uint32_t *s_ctl = reinterpret_cast<uint32_t *>(s_excl + MAX_SCAN);                        // [0] tile

    // one-time: program + column table into shared memory
    for (uint32_t i = tid; i < P.n_instr * (sizeof(DInstr) / 16); i += NT)
        reinterpret_cast<uint4 *>(s_prog)[i] = reinterpret_cast<const uint4 *>(P.prog)[i];
    for (uint32_t i = tid; i < P.n_in * (sizeof(ColIn) / 8); i += NT)
        reinterpret_cast<uint64_t *>(s_cols)[i] = reinterpret_cast<const uint64_t *>(P.in)[i];

    VMThread t;
    t.scr_cap = P.scratch_per_thread;
    t.scratch = P.scratch + ((size_t)blockIdx.x * NT + tid) * (size_t)P.scratch_per_thread;

    const uint32_t state_stride = 1 + 2 * K;
    // work size: known to the host, or (dense launch behind a prefilter that was not waited for) read from the device and clamped to
    // the capacity everything was sized for; a count beyond the capacity raises flag 8 and the host redoes the launch
    uint64_t n_work = P.n_work;
    uint32_t n_tiles = P.n_tiles;
    if (P.n_work_dev) {
        const uint64_t actual = *P.n_work_dev;
        if (actual > P.n_work && blockIdx.x == 0 && tid == 0) atomicOr(&P.counters[1], 8u);
        n_work = actual < P.n_work ? actual : P.n_work;
        n_tiles = (uint32_t)((n_work + T - 1) / T);
        if (n_tiles == 0 && blockIdx.x == 0 && tid == 0)
            for (uint32_t c = 0; c < P.n_out; ++c)
                if (P.out[c].strk >= 0) P.out[c].offsets[0] = 0;
    }

    while (true) {
        __syncthreads();
        if (tid == 0) {
            s_ctl[0] = atomicAdd(&P.counters[0], 1u);
            s_ctl[1] = 0;
        }
        for (uint32_t i = tid; i < 2 * W; i += NT) keep_bits[i] = 0;  // keep_bits and exc_bits
        __syncthreads();
        const uint32_t tile = s_ctl[0];
        if (tile >= n_tiles) break;
        const uint64_t base = (uint64_t)tile * T;  // position in the work list (== input row without a rowlist)
        t.scr_used = 0;

        // ---- evaluate -----------------------------------------------------------------------
        auto stage_row = [&](uint32_t lr) {
            for (uint32_t c = 0; c < P.n_out; ++c) {
                const OutCol &oc = P.out[c];
                if (oc.strk >= 0) {
                    uint64_t *st = reinterpret_cast<uint64_t *>(s_stage + oc.stage_off) + 2 * (size_t)lr;
                    st[0] = VM<NT>::R(s_regs, oc.slot * VM<NT>::SLOT_BYTES);
                    st[1] = VM<NT>::R(s_regs, (oc.slot + 1) * VM<NT>::SLOT_BYTES);
                } else {
                    reinterpret_cast<uint64_t *>(s_stage + oc.stage_off)[lr] = VM<NT>::R(s_regs, oc.slot * VM<NT>::SLOT_BYTES);
                }
            }
        };

        for (uint32_t s = 0; s < R; ++s) {
            const uint32_t lr = s * NT + tid;
            const uint64_t w = base + lr;
            const bool valid = w < n_work;
            const uint64_t row = P.rowlist ? (valid ? P.rowlist[w] : 0) : w;
            t.alive = valid;
            t.exc_code = 0;
            TPLX_VM_RUN(s_prog, P.n_instr, s_regs, s_cols, row, w, P.cpool, t);
            const bool exc = t.exc_code != 0;
            const uint32_t kb = __ballot_sync(0xFFFFFFFFu, t.alive);
            const uint32_t eb = __ballot_sync(0xFFFFFFFFu, exc);
            if (lane == 0) { keep_bits[lr >> 5] = kb; exc_bits[lr >> 5] = eb; }
            if (t.alive && !P.inplace) stage_row(lr);
            if (exc) {
                exc_stage[lr * exc_stride] = t.exc_code | (t.exc_op << 16);

            }
        }
        __syncthreads();

        rows_tile_finish(P, TileSmem{s_stage, s_regs, s_stash, keep_bits, exc_bits, keep_pre, exc_pre, exc_stage, exc_stride, s_vals, s_excl}, tile, base,
                         R, T, W, K, state_stride, n_tiles);
    }
}
#endif  // K1

// =============================================================================================
// K3: rows in -> aggregate (fixed reduction tree; see DESIGN.md "reduction tree")
//   thread t of a tile folds local rows t, t+NT, ... in order from the identity,
//   warp tree via shfl_down 16,8,4,2,1, warps combined sequentially -> tile partial.
// =============================================================================================
#if !defined(TPLX_JIT) || TPLX_JIT_KIND == 4
#ifdef TPLX_JIT
extern "C" __global__ void __launch_bounds__(NT, TPLX_JIT_MIN_CTAS) tplx_jit_kernel(const KParams *__restrict__ Pg) {
#else
__global__ void __launch_bounds__(NT) stage_agg_kernel(const KParams *__restrict__ Pg) {
#endif
    extern __shared__ __align__(16) uint8_t smem[];
    const KParams &P = *Pg;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t R = P.R, T = R * NT;

    DInstr *s_prog = reinterpret_cast<DInstr *>(smem);
    ColIn *s_cols = reinterpret_cast<ColIn *>(smem + P.smem_cols_off);
    uint8_t *s_regs = smem + P.smem_regs_off + tid * 8;  // this thread's register column
    uint64_t *s_wacc = reinterpret_cast<uint64_t *>(smem + P.smem_misc_off);  // [NT/32][n_accs]

    for (uint32_t i = tid; i < P.n_instr * (sizeof(DInstr) / 16); i += NT)
        reinterpret_cast<uint4 *>(s_prog)[i] = reinterpret_cast<const uint4 *>(P.prog)[i];
    for (uint32_t i = tid; i < P.n_in * (sizeof(ColIn) / 8); i += NT)
        reinterpret_cast<uint64_t *>(s_cols)[i] = reinterpret_cast<const uint64_t *>(P.in)[i];
    __syncthreads();

    VMThread t;
    t.scr_cap = P.scratch_per_thread;
    t.scratch = P.scratch + ((size_t)blockIdx.x * NT + tid) * (size_t)P.scratch_per_thread;
    const uint32_t na = P.n_accs;

    for (uint32_t tile = blockIdx.x; tile < P.n_tiles; tile += gridDim.x) {
        const uint64_t base = (uint64_t)tile * T;
        uint64_t acc[TPLX_MAX_ACCS];
#pragma unroll
        for (uint32_t k = 0; k < TPLX_MAX_ACCS; ++k) acc[k] = k < na ? acc_identity(P.accs[k].kind) : 0;
        for (uint32_t s = 0; s < R; ++s) {
            const uint64_t row = base + (uint64_t)s * NT + tid;
            t.alive = row < P.n_rows;
            t.exc_code = 0;
            t.scr_used = 0;
            TPLX_VM_RUN(s_prog, P.n_instr, s_regs, s_cols, row, row, P.cpool, t);
            if (t.alive) {
#pragma unroll
                for (uint32_t k = 0; k < TPLX_MAX_ACCS; ++k)
                    if (k < na) acc[k] = acc_combine(P.accs[k].kind, acc[k], VM<NT>::R(s_regs, P.accs[k].slot * VM<NT>::SLOT_BYTES));
            }
            if (t.exc_code) {
                uint32_t pos = atomicAdd(&P.counters[2], 1u);
                if (pos < P.cap_exc) {
                    tplx_exception_rec rec;
                    rec.row = (int64_t)row;
                    rec.row_no = 0;  // assigned on the host after sorting by row
                    rec.code = t.exc_code;
                    rec.op_id = P.opids[t.exc_op];
                    P.exc[pos] = rec;
                } else atomicOr(&P.counters[1], 4u);
            }
        }
        // warp tree: shfl_down 16,8,4,2,1 (lane 0 holds the warp partial)
#pragma unroll
        for (uint32_t k = 0; k < TPLX_MAX_ACCS; ++k) {
            if (k < na) {
                uint64_t v = acc[k];
#pragma unroll
                for (int o = 16; o; o >>= 1) {
                    uint64_t other = __shfl_down_sync(0xFFFFFFFFu, v, o);
                    v = acc_combine(P.accs[k].kind, v, other);
                }
                if (lane == 0) s_wacc[warp * na + k] = v;
            }
        }
        __syncthreads();
        if (tid < na) {
            uint64_t v = s_wacc[tid];
            for (uint32_t w = 1; w < NT / 32; ++w) v = acc_combine(P.accs[tid].kind, v, s_wacc[w * na + tid]);
            P.tile_partials[(size_t)tile * na + tid] = v;
        }
        __syncthreads();
    }
}

#endif  // K3

#ifndef TPLX_JIT
// thread t folds tile partials t, t+FIN_NT, ... in order; warp tree; warps sequential; then init (+) total
__global__ void __launch_bounds__(FIN_NT) agg_finalize_kernel(const KParams *__restrict__ Pg) {
    __shared__ uint64_t s_w[FIN_NT / 32];
    const KParams &P = *Pg;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (uint32_t k = 0; k < P.n_accs; ++k) {
        const uint32_t kind = P.accs[k].kind;
        uint64_t v = acc_identity(kind);
        for (uint32_t tile = tid; tile < P.n_tiles; tile += FIN_NT)
            v = acc_combine(kind, v, P.tile_partials[(size_t)tile * P.n_accs + k]);
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            uint64_t other = __shfl_down_sync(0xFFFFFFFFu, v, o);
            v = acc_combine(kind, v, other);
        }
        if (lane == 0) s_w[warp] = v;
        __syncthreads();
        if (tid == 0) {
            uint64_t tot = s_w[0];
            for (uint32_t w = 1; w < FIN_NT / 32; ++w) tot = acc_combine(kind, tot, s_w[w]);
            // per-task intermediate starts from the initial value (BlockBasedTaskBuilder.cc:185-206)
            P.agg_out[k] = acc_combine(kind, (uint64_t)P.accs[k].init, tot);
        }
        __syncthreads();
    }
}
#endif  // !TPLX_JIT

}  // namespace tplx
