// vecvm.cuh — K1v: the row kernel for stages made of fixed-width columns only (BASELINE config 0 / C1 and every numeric
// map / filter / project pipeline): the closed-form fast path the reference gets from specialising its block loop per stage
// (tuplex/core/src/physical/TuplexSourceTaskBuilder.cc:104-215 + PipelineBuilder.cc:565-700 for fixed-width rows).
//
// Same op program, same per-row semantics as vm.cuh (every op is the same single integer / IEEE operation), evaluated
// VECTOR-AT-A-TIME: a thread owns V = 2J rows of a tile; one instruction dispatch (uniform fetch + jump table) is followed by 2J
// row operations, so the interpretive overhead per row shrinks by 2J. Mapping onto the SM:
//   * inputs: coalesced 128-bit global loads (LDG.E.128: thread t reads rows 2t, 2t+1 of every 512-row slab of the tile);
//   * ACCUMULATOR CHAINS: the host's vector planner (vec_plan in tplx_gpu.cu) finds the straight-line producer -> consumer pairs of
//     the program; the consumer takes the value from the thread's registers (the accumulator = result of the previous micro-op)
//     and a result nobody else reads is never stored. compare + filter and (x mod 2^k) + compare are single micro-ops.
//     C1 (x*x, x % 2 == 0) runs as LDCOL -> IMUL -> masked-compare-filter: one LDG.128 and one STS.128 per two rows;
//   * what does have to live across micro-ops sits in shared memory as regs[slot][local row] — one conflict-free LDS.128 /
//     STS.128 moves two rows, and because a slot is indexed by the local row it IS the staging array of an output column;
//   * compaction by the OWNER of a row: two ballots per 512-row slab give every thread the rank of its rows inside the warp,
//     one 32-entry scan of (slab, warp) counts gives the rank inside the tile, a block-wide packed look-back (below) the
//     rank in the output — the thread then stores its own rows (dense, ascending addresses across the warp). No bitmaps.
// Strings never enter this kernel (the host selects it only for programs without string values).
#pragma once
#include <stdint.h>
#include "kernels.cuh"

namespace tplx {

// Vector micro-ops: produced by the host's planner from the IR ops, never part of the IR. Dense numbering.
// V_ISHRK / V_IANDK: strength-reduced x // 2^k, x % 2^k (floored semantics make both exact for every dividend).
enum VOp : uint32_t {
    V_NOP = 0, V_LDCOL, V_LDI, V_LDROW, V_MOV, V_SEL,
    V_IADD, V_ISUB, V_IMUL, V_INEG, V_IAND, V_IOR, V_IXOR, V_ISHL, V_ISHR, V_ISHRK, V_IANDK, V_IABS,
    V_FADD, V_FSUB, V_FMUL, V_FNEG, V_FABS, V_I2F, V_F2I, V_BAND, V_BOR, V_BNOT,
    V_ICMP_EQ, V_ICMP_NE, V_ICMP_LT, V_ICMP_LE, V_ICMP_GT, V_ICMP_GE,
    V_FCMP_EQ, V_FCMP_NE, V_FCMP_LT, V_FCMP_LE, V_FCMP_GT, V_FCMP_GE,
    V_IFLOORDIV, V_IMOD, V_FDIV, V_FMOD, V_FFLOORDIV, V_FILTER, V_RAISE, V_COUNT
};
// planner flags of a micro-op
enum VFlag : uint32_t {
    VX_A_ACC = 1,     // operand a = the accumulator (result of the previous micro-op) instead of a slot
    VX_B_ACC = 2,     // operand b likewise (only together with VX_A_ACC: loading a would overwrite the accumulator)
    VX_NOSTORE = 4,   // nobody reads the result from its slot: keep it in the accumulator only
    VX_FILTER = 8,    // boolean result: rows with 0 leave the pipeline (the FILTER that followed, fused)
    VX_A_MASK = 16,   // integer compares: a <- a & imm2 first (the x % 2^k that preceded, fused)
    // set by the encoder (vec_encode), not by the planner:
    VX_LOAD_A = 32,   // the op reads a and it is not in the accumulator: load it first
    VX_RESULT = 64,   // the op produces a value (everything but FILTER / RAISE)
    VX_A_THREAD = 128,  // operand a is a slot (per-thread address, stride SLAB); clear = a constant pair inside the instruction
    VX_B_THREAD = 256,  // operand b likewise
};

// Device format of a micro-op: operands are ADDRESSES, so that a slot and a constant are read by the same 128-bit shared-memory
// load (a constant is a pair [v, v] inside the instruction itself, read by all lanes at once: stride 0, no per-thread offset).
struct __align__(16) VInstr {
    uint32_t op_opidx;  // vop | opidx << 16
    uint32_t xf;        // VFlag bits
    uint32_t dst;       // byte offset of the destination slot from the start of the register file, NOOFF = none
    uint32_t guard;     // likewise, NOOFF = unguarded
    uint32_t pa, pb;    // operands a, b: byte offset from the start of shared memory (slot: its first row; constant: the pair below)
    uint32_t pc;        // operand c (SEL condition): byte offset of its slot from the start of the register file
    uint32_t pad;
    uint64_t kb[2];     // [imm, imm]: constant b; scalar immediates (column index, shift count, exception code)
    uint64_t ka[2];     // [imm2, imm2]: constant a, or the mask of VX_A_MASK
};
static_assert(sizeof(VInstr) == 64, "VInstr layout");

template <int J>
struct VecVM {
    static constexpr uint32_t V = 2 * J;                 // rows per thread
    static constexpr uint32_t T = V * NT;                // rows per tile
    static constexpr uint32_t SLAB = NT * 16;            // bytes between the two-row groups j and j+1 of one slot
    static constexpr uint32_t SLOT_BYTES = T * 8;        // one slot = T values indexed by local row

    struct State {
        uint32_t alive;  // bit v: row v of this thread is still in the pipeline
        uint32_t exc;    // bit v: row v raised
    };
    // local row of (j, b) for this thread: lr = j * 2 NT + 2 tid + b
    static __device__ __forceinline__ uint32_t lrow(uint32_t j, uint32_t b) { return j * 2 * NT + 2 * threadIdx.x + b; }

    static __device__ __forceinline__ ulonglong2 ld2(const uint8_t *rb, uint32_t off, uint32_t j) {
        return *reinterpret_cast<const ulonglong2 *>(rb + off + j * SLAB);
    }
    static __device__ __forceinline__ void st2(uint8_t *rb, uint32_t off, uint32_t j, ulonglong2 v) {
        *reinterpret_cast<ulonglong2 *>(rb + off + j * SLAB) = v;
    }
    static __device__ __forceinline__ void raise_row(State &st, uint32_t v, uint32_t code, uint32_t opidx, uint32_t *exc_stage, uint32_t lr) {
        st.alive &= ~(1u << v);
        st.exc |= 1u << v;
        exc_stage[lr] = code | (opidx << 16);
    }

    // smem = start of shared memory (operand addresses), rb = register file + tid * 16. tile_row0 = first input row of the tile;
    // full = the tile has T rows (uniform).
    static __device__ void run(const VInstr *__restrict__ prog, uint32_t n_instr, const uint8_t *__restrict__ smem, uint8_t *__restrict__ rb,
                               const ColIn *__restrict__ cols, uint64_t tile_row0, uint64_t n_rows, bool full, State &st,
                               uint32_t *__restrict__ exc_stage) {
        const uint32_t tid16 = threadIdx.x * 16;
        ulonglong2 acc[J];  // the accumulator: operand a on entry to an op, its result on exit
#pragma unroll
        for (uint32_t j = 0; j < J; ++j) acc[j] = make_ulonglong2(0, 0);
        for (uint32_t pc = 0; pc < n_instr; ++pc) {
            const uint4 w0 = *reinterpret_cast<const uint4 *>(&prog[pc]);
            const uint4 w1 = *reinterpret_cast<const uint4 *>(&prog[pc].pa);
            const uint32_t op = w0.x & 0xFFFF, opidx = w0.x >> 16, xf = w0.y, dst = w0.z, guard = w0.w;
            uint32_t act = st.alive;  // rows this instruction executes for
            const bool guarded = guard != NOOFF;
            if (guarded) {
#pragma unroll
                for (uint32_t j = 0; j < J; ++j) {
                    const ulonglong2 g = ld2(rb, guard, j);
                    if (g.x == 0) act &= ~(1u << (2 * j));
                    if (g.y == 0) act &= ~(2u << (2 * j));
                }
                if (!__any_sync(0xFFFFFFFFu, act != 0)) continue;  // untaken branch: the warp skips the op
            }
            if (xf & VX_LOAD_A) {
                const uint8_t *pA = smem + w1.x + ((xf & VX_A_THREAD) ? tid16 : 0u);
                const uint32_t sA = (xf & VX_A_THREAD) ? SLAB : 0u;
#pragma unroll
                for (uint32_t j = 0; j < J; ++j) acc[j] = *reinterpret_cast<const ulonglong2 *>(pA + j * sA);
            }
            const uint8_t *pB = smem + w1.y + ((xf & VX_B_THREAD) ? tid16 : 0u);
            const uint32_t sB = (xf & VX_B_THREAD) ? SLAB : 0u;
#define LB(j) (*reinterpret_cast<const ulonglong2 *>(pB + (j) * sB))
            // binary op on (accumulator, b): b is the accumulator itself (x * x), or one 128-bit load per two rows
#define BIN(EXPR)                                                                          \
    if (xf & VX_B_ACC) {                                                                   \
        _Pragma("unroll") for (uint32_t j = 0; j < J; ++j) {                               \
            { const uint64_t x = acc[j].x, y = x; acc[j].x = (uint64_t)(EXPR); }           \
            { const uint64_t x = acc[j].y, y = x; acc[j].y = (uint64_t)(EXPR); }           \
        }                                                                                  \
    } else {                                                                               \
        _Pragma("unroll") for (uint32_t j = 0; j < J; ++j) {                               \
            const ulonglong2 B = LB(j);                                                    \
            { const uint64_t x = acc[j].x, y = B.x; acc[j].x = (uint64_t)(EXPR); }         \
            { const uint64_t x = acc[j].y, y = B.y; acc[j].y = (uint64_t)(EXPR); }         \
        }                                                                                  \
    }                                                                                      \
    break
#define UNA(EXPR)                                                                          \
    _Pragma("unroll") for (uint32_t j = 0; j < J; ++j) {                                   \
        { const uint64_t x = acc[j].x; acc[j].x = (uint64_t)(EXPR); }                      \
        { const uint64_t x = acc[j].y; acc[j].y = (uint64_t)(EXPR); }                      \
    }                                                                                      \
    break
            // integer compares: optionally on (a & mask) — the x % 2^k that preceded
#define ICMP(EXPR)                                                                         \
    {                                                                                      \
        const uint64_t msk = (xf & VX_A_MASK) ? prog[pc].ka[0] : ~0ull;                    \
        _Pragma("unroll") for (uint32_t j = 0; j < J; ++j) {                               \
            const ulonglong2 B = (xf & VX_B_ACC) ? acc[j] : LB(j);                         \
            { const int64_t x = (int64_t)(acc[j].x & msk), y = (int64_t)B.x; acc[j].x = (uint64_t)(EXPR); } \
            { const int64_t x = (int64_t)(acc[j].y & msk), y = (int64_t)B.y; acc[j].y = (uint64_t)(EXPR); } \
        }                                                                                  \
    }                                                                                      \
    break
#define F(x) __longlong_as_double((long long)(x))
#define U(d) ((uint64_t)__double_as_longlong(d))
            // ops that can raise: row by row for the active rows only; a raising row leaves the pipeline
#define RAISING(...)                                                                       \
    _Pragma("unroll") for (uint32_t v = 0; v < V; ++v) {                                   \
        if (!((act >> v) & 1u)) continue;                                                  \
        const ulonglong2 Bv = LB(v >> 1);                                                  \
        const uint64_t x = (v & 1) ? acc[v >> 1].y : acc[v >> 1].x, y = (v & 1) ? Bv.y : Bv.x; \
        uint64_t r = 0;                                                                    \
        bool bad = false;                                                                  \
        __VA_ARGS__;                                                                       \
        if (bad) raise_row(st, v, TPLX_EC_ZERODIVISIONERROR, opidx, exc_stage, lrow(v >> 1, v & 1)); \
        if (v & 1) acc[v >> 1].y = r; else acc[v >> 1].x = r;                              \
    }                                                                                      \
    break
            switch (op) {
                case V_LDCOL: {
                    const uint64_t *src = reinterpret_cast<const uint64_t *>(cols[prog[pc].kb[0]].data);
#ifdef __CUDA_ARCH__
                    __builtin_assume(__isGlobal(src));
#endif
#pragma unroll
                    for (uint32_t j = 0; j < J; ++j) {
                        const uint64_t row = tile_row0 + lrow(j, 0);
                        ulonglong2 v = make_ulonglong2(0, 0);
                        if (full || row + 1 < n_rows) v = *reinterpret_cast<const ulonglong2 *>(src + row);  // 16-byte aligned: row is even, base is
                        else if (row < n_rows) v.x = src[row];
                        acc[j] = v;
                    }
                    break;
                }
                case V_LDI: {
                    const uint64_t imm = prog[pc].kb[0];
#pragma unroll
                    for (uint32_t j = 0; j < J; ++j) acc[j] = make_ulonglong2(imm, imm);
                    break;
                }
                case V_LDROW:
#pragma unroll
                    for (uint32_t j = 0; j < J; ++j) {
                        const uint64_t row = tile_row0 + lrow(j, 0);
                        acc[j] = make_ulonglong2(row, row + 1);
                    }
                    break;
                case V_MOV: break;  // a is already in the accumulator
                case V_SEL:
#pragma unroll
                    for (uint32_t j = 0; j < J; ++j) {
                        const ulonglong2 B = (xf & VX_B_ACC) ? acc[j] : LB(j), Cn = ld2(rb, w1.z, j);
                        if (!Cn.x) acc[j].x = B.x;
                        if (!Cn.y) acc[j].y = B.y;
                    }
                    break;
                case V_IADD: BIN(x + y);
                case V_ISUB: BIN(x - y);
                case V_IMUL: BIN(x * y);
                case V_INEG: UNA((uint64_t)0 - x);
                case V_IAND: BIN(x & y);
                case V_IOR: BIN(x | y);
                case V_IXOR: BIN(x ^ y);
                case V_ISHL: BIN(x << (y & 63));
                case V_ISHR: BIN((uint64_t)((int64_t)x >> (y & 63)));
                case V_ISHRK: { const uint32_t k = (uint32_t)prog[pc].kb[0] & 63; UNA((uint64_t)((int64_t)x >> k)); }
                case V_IANDK: { const uint64_t m = prog[pc].kb[0]; UNA(x & m); }
                case V_IABS: UNA((int64_t)x < 0 ? (uint64_t)0 - x : x);
                case V_FADD: BIN(U(__dadd_rn(F(x), F(y))));
                case V_FSUB: BIN(U(__dsub_rn(F(x), F(y))));
                case V_FMUL: BIN(U(__dmul_rn(F(x), F(y))));
                case V_FNEG: UNA(x ^ 0x8000000000000000ull);
                case V_FABS: UNA(x & 0x7FFFFFFFFFFFFFFFull);
                case V_I2F: UNA(U((double)(int64_t)x));
                case V_F2I: UNA((uint64_t)(int64_t)F(x));
                case V_BAND: BIN((x != 0) & (y != 0));
                case V_BOR: BIN((x != 0) | (y != 0));
                case V_BNOT: UNA(x == 0);
                case V_ICMP_EQ: ICMP(x == y);
                case V_ICMP_NE: ICMP(x != y);
                case V_ICMP_LT: ICMP(x < y);
                case V_ICMP_LE: ICMP(x <= y);
                case V_ICMP_GT: ICMP(x > y);
                case V_ICMP_GE: ICMP(x >= y);
                // ordered predicates: false when either side is NaN
                case V_FCMP_EQ: BIN(F(x) == F(y));
                case V_FCMP_NE: BIN((F(x) < F(y)) || (F(x) > F(y)));
                case V_FCMP_LT: BIN(F(x) < F(y));
                case V_FCMP_LE: BIN(F(x) <= F(y));
                case V_FCMP_GT: BIN(F(x) > F(y));
                case V_FCMP_GE: BIN(F(x) >= F(y));
                case V_IFLOORDIV: RAISING({ if ((int64_t)y == 0) bad = true; else r = (uint64_t)floordiv_i64((int64_t)x, (int64_t)y); });
                case V_IMOD: RAISING({ if ((int64_t)y == 0) bad = true; else r = (uint64_t)floormod_i64((int64_t)x, (int64_t)y); });
                case V_FDIV: RAISING({ if (F(y) == 0.0) bad = true; else r = U(__ddiv_rn(F(x), F(y))); });
                case V_FMOD: RAISING({
                    if (F(y) == 0.0) bad = true;
                    else {
                        double m = fmod(F(x), F(y));  // == LLVM frem, exact
                        if (m != 0.0 && ((m < 0.0) != (F(y) < 0.0))) m = __dadd_rn(m, F(y));
                        r = U(m);
                    }
                });
                case V_FFLOORDIV: RAISING({
                    const int64_t xi = (int64_t)F(x), yi = (int64_t)F(y);
                    if (F(y) == 0.0 || yi == 0) bad = true;
                    else r = U((double)floordiv_i64(xi, yi));
                });
                case V_FILTER:
#pragma unroll
                    for (uint32_t j = 0; j < J; ++j) {
                        if (acc[j].x == 0) st.alive &= ~(act & (1u << (2 * j)));
                        if (acc[j].y == 0) st.alive &= ~(act & (2u << (2 * j)));
                    }
                    if (!__any_sync(0xFFFFFFFFu, st.alive != 0)) return;  // the warp is empty: nothing that follows can execute
                    break;
                case V_RAISE: {
                    const uint32_t code = (uint32_t)prog[pc].kb[0];
#pragma unroll
                    for (uint32_t v = 0; v < V; ++v)
                        if ((act >> v) & 1u) raise_row(st, v, code, opidx, exc_stage, lrow(v >> 1, v & 1));
                    break;
                }
                default: break;
            }
#undef LB
#undef BIN
#undef UNA
#undef ICMP
#undef F
#undef U
#undef RAISING
            // ---- result: merge under a guard, store unless nobody reads the slot, filter ----
            if (xf & VX_RESULT) {
                if (guarded) {  // rows outside the guard keep the old destination (phi of an if-converted branch)
#pragma unroll
                    for (uint32_t j = 0; j < J; ++j) {
                        const ulonglong2 o = ld2(rb, dst, j);
                        if (!((act >> (2 * j)) & 1u)) acc[j].x = o.x;
                        if (!((act >> (2 * j + 1)) & 1u)) acc[j].y = o.y;
                    }
                }
                if (!(xf & VX_NOSTORE)) {
#pragma unroll
                    for (uint32_t j = 0; j < J; ++j) st2(rb, dst, j, acc[j]);
                }
                if (xf & VX_FILTER) {  // unguarded (planner): act == alive
#pragma unroll
                    for (uint32_t j = 0; j < J; ++j) {
                        if (acc[j].x == 0) st.alive &= ~(1u << (2 * j));
                        if (acc[j].y == 0) st.alive &= ~(2u << (2 * j));
                    }
                    if (!__any_sync(0xFFFFFFFFu, st.alive != 0)) return;
                }
            }
        }
    }
};

// ---- tile tail: ranks by the owner, block-wide decoupled look-back, dense write (fixed-width outputs only) ---------------------
// The scalar kernel's look-back (rows_tile_finish: one warp, a 32-tile window per round, K values behind a status flag and a fence)
// is fine for heavy tiles; a fixed-width tile is evaluated in ~1-2 us, and then the speed at which inclusive prefixes propagate
// (32 tiles per L2 round trip) bounds the whole kernel. Here a tile's scan state is ONE 64-bit word
//   [status:2 | rows kept:31 | exception rows:31]   status 1 = this tile's counts, 2 = inclusive prefix
// written with a single relaxed store (no fence: status and values travel together), and ALL 256 threads look back at once: thread t
// polls tile - 1 - t, the block adds the counts up to the nearest inclusive word — 256 tiles per round trip.
__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// Block-wide decoupled look-back of a tile (all NT threads call it): on return pre_keep / pre_exc = rows kept / raised by every earlier
// tile, and this tile's inclusive prefix has been published. s_scr: 4 * NT/32 words of shared memory (double-buffered per round).
__device__ __forceinline__ void vec_lookback(const KParams &P, uint32_t tile, uint32_t n_keep, uint32_t n_exc, uint64_t *s_scr, uint64_t &pre_keep,
                                             uint64_t &pre_exc) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tile > 0) {
        int64_t p = (int64_t)tile - 1;
        for (uint32_t round = 0;; ++round) {
            uint64_t *scr = s_scr + (round & 1u) * (2 * (NT / 32));  // double-buffered: one barrier per round
            const int64_t q = p - (int64_t)tid;
            uint64_t wd = (uint64_t)2 << 62;  // tiles before the first count as an inclusive prefix of zero
            if (q >= 0) do { wd = ld_relaxed_u64(P.tile_state + q); } while ((wd >> 62) == 0);
            const bool incl = (wd >> 62) == 2;
            const uint32_t im = __ballot_sync(0xFFFFFFFFu, incl);
            const uint32_t first = im ? (uint32_t)(__ffs(im) - 1) : 32u;  // nearest inclusive word inside this warp's 32 tiles
            uint64_t k = lane <= first ? (wd >> 31) & 0x7FFFFFFFull : 0, e = lane <= first ? wd & 0x7FFFFFFFull : 0;
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                k += __shfl_xor_sync(0xFFFFFFFFu, k, o);
                e += __shfl_xor_sync(0xFFFFFFFFu, e, o);
            }
            if (lane == 0) {
                scr[warp * 2] = (k << 32) | e;  // counts are < 2^31 in total: 32 bits each
                scr[warp * 2 + 1] = im ? 1 : 0;
            }
            __syncthreads();
            bool done = false;
            for (uint32_t w = 0; w < NT / 32 && !done; ++w) {  // warps cover tile-1-32w .. : nearest first
                pre_keep += scr[w * 2] >> 32;
                pre_exc += scr[w * 2] & 0xFFFFFFFFull;
                done = scr[w * 2 + 1] != 0;
            }
            if (done) break;
            p -= NT;
        }
        if (tid == 0) st_cg_u64(P.tile_state + tile, ((uint64_t)2 << 62) | ((pre_keep + n_keep) << 31) | (pre_exc + n_exc));
    }
}

// K1v kernel: persistent CTAs, ticketed tiles of T = 2J * 256 rows.
// Shared memory: prog (VInstr) | cols | regs (n_slots x T x 8 B; output columns are staged in place) | misc: s_cnt[8J] exc_stage[T]
// scan scratch, tickets.
// Row order inside a tile: slab j (512 rows), warp w (64 rows), lane (2 rows). s_cnt[j * 8 + w] = kept | raised << 16 of that group.
#ifdef TPLX_JIT
// Specialised evaluation (stage specialiser, jit.inl): per two-row group one LDG.128 per used input column, the generated
// straight-line row function for each of the two rows (slots in registers), one STS.128 per live-out slot into the compact
// register file the tile tail reads. Same State / exc_stage protocol as VecVM::run.
template <int J>
__device__ __forceinline__ void jit_load_vec(ulonglong2 (&vin)[J][JIT_NIN], const ColIn *__restrict__ cols, uint64_t tile_row0, uint64_t n_rows, bool full) {
#pragma unroll
    for (uint32_t k = 0; k < JIT_NIN; ++k) {
        const uint64_t *src = reinterpret_cast<const uint64_t *>(cols[jit_incol(k)].data);
        __builtin_assume(__isGlobal(src));
#pragma unroll
        for (uint32_t j = 0; j < J; ++j) {
            const uint64_t row = tile_row0 + VecVM<J>::lrow(j, 0);
            ulonglong2 v = make_ulonglong2(0, 0);
            if (full || row + 1 < n_rows) v = *reinterpret_cast<const ulonglong2 *>(src + row);  // 16-byte aligned: row is even, base is
            else if (row < n_rows) v.x = src[row];
            vin[j][k] = v;
        }
    }
}
template <int J>
__device__ __forceinline__ void jit_eval_vec(const ulonglong2 (&vin)[J][JIT_NIN], uint8_t *__restrict__ rb, uint64_t tile_row0, typename VecVM<J>::State &st,
                                             uint32_t *__restrict__ exc_stage) {
#pragma unroll
    for (uint32_t j = 0; j < J; ++j) {
        const uint64_t row = tile_row0 + VecVM<J>::lrow(j, 0);
        uint64_t in0[JIT_NIN], in1[JIT_NIN], o0[JIT_NLIVE], o1[JIT_NLIVE];
#pragma unroll
        for (uint32_t k = 0; k < JIT_NIN; ++k) { in0[k] = vin[j][k].x; in1[k] = vin[j][k].y; }
#pragma unroll
        for (uint32_t k = 0; k < JIT_NLIVE; ++k) { o0[k] = 0; o1[k] = 0; }
        bool a0 = (st.alive >> (2 * j)) & 1u, a1 = (st.alive >> (2 * j + 1)) & 1u;
        uint32_t e0 = 0, e1 = 0;
        if (a0) jit_row_fixed(row, in0, a0, e0, o0);
        if (a1) jit_row_fixed(row + 1, in1, a1, e1, o1);
        if (!a0) st.alive &= ~(1u << (2 * j));
        if (!a1) st.alive &= ~(2u << (2 * j));
        if (e0) VecVM<J>::raise_row(st, 2 * j, e0 & 0xFFFFu, e0 >> 16, exc_stage, VecVM<J>::lrow(j, 0));
        if (e1) VecVM<J>::raise_row(st, 2 * j + 1, e1 & 0xFFFFu, e1 >> 16, exc_stage, VecVM<J>::lrow(j, 1));
#pragma unroll
        for (uint32_t k = 0; k < JIT_NLIVE; ++k) VecVM<J>::st2(rb, k * VecVM<J>::SLOT_BYTES, j, make_ulonglong2(o0[k], o1[k]));
    }
}
#endif

#if defined(TPLX_JIT) && TPLX_JIT_KIND == 6
// ---- K1w: the specialised fixed-width row kernel with WIDE tiles ---------------------------------------------------------------------
// On C1, with the interpretation gone, K1v is bound by the latency chain of a tile — ticket, LDG,
// counts, look-back over every earlier tile still in flight, stores — of which the look-back waits for the SLOWEST load among all
// predecessors (in-order retirement over a window of ~1000 tiles), however few instructions the tile takes.
// Only resident warps hide that, and a specialised row function leaves registers and shared memory to spare. So a CTA takes B = 4
// sub-batches of 2048 rows per ticket: one ticket, one count barrier, ONE look-back and one inclusive-prefix publication per 8192 rows,
// 64 KB of loads per CTA between two waits; the sub-batches are evaluated back to back (the LDG.128s of sub-batch b + 1 are issued before
// sub-batch b is evaluated when the registers allow), their live-out slots staged side by side in the compact register file
// (regs[slot][b][local row]), exception codes of raising rows in slot 0 of that row (a raising row is not written).
// Same row order, same packed tile-state word, same output as K1v with tiles four times the size.
extern "C" __global__ void __launch_bounds__(NT, TPLX_JIT_MIN_CTAS) tplx_jit_kernel(const __grid_constant__ KParams P) {
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr int J = 4, B = 4;
    using VV = VecVM<J>;
    constexpr uint32_t TS = VV::T, T = B * TS, SLOT_W = T * 8;  // rows per sub-batch / per tile, bytes of one slot of the wide register file
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    ColIn *s_cols = reinterpret_cast<ColIn *>(smem + P.smem_cols_off);
    uint8_t *s_regs = smem + P.smem_regs_off;
    uint32_t *s_cnt = reinterpret_cast<uint32_t *>(smem + P.smem_misc_off);  // [B][32]: kept | raised << 16 per (sub-batch, slab, warp)
    uint64_t *s_scr = reinterpret_cast<uint64_t *>(s_cnt + B * 32);
    uint32_t *s_ctl = reinterpret_cast<uint32_t *>(s_scr + 4 * (NT / 32));

    for (uint32_t i = tid; i < P.n_in * (sizeof(ColIn) / 8); i += NT)
        reinterpret_cast<uint64_t *>(s_cols)[i] = reinterpret_cast<const uint64_t *>(P.in)[i];
    uint8_t *rb = s_regs + tid * 16;
    const uint32_t lt = (1u << lane) - 1u;
    auto code_at = [&](uint32_t b, uint32_t lr) -> uint32_t * {  // code | opidx << 16 of a raising row: the low word of its slot 0
        return reinterpret_cast<uint32_t *>(s_regs + ((size_t)b * TS + lr) * 8);
    };

    if (tid == 0) s_ctl[0] = atomicAdd(&P.counters[0], 1u);
    while (true) {
        __syncthreads();  // the ticket is visible; s_cnt and the look-back scratch of the previous tile are no longer read
        const uint32_t tile = s_ctl[0];
        if (tile >= P.n_tiles) break;
        const uint64_t base = (uint64_t)tile * T;

        // ---- evaluate the B sub-batches ----
        uint32_t alive[B], excb[B];
        auto eval = [&](uint32_t b, const ulonglong2 (&vin)[J][JIT_NIN]) {
            const uint64_t sb = base + (uint64_t)b * TS;
            uint32_t al = 0, ex = 0;
            uint32_t ec[2 * J];
#pragma unroll
            for (uint32_t j = 0; j < J; ++j) {
                const uint64_t row = sb + VV::lrow(j, 0);
                uint64_t in0[JIT_NIN], in1[JIT_NIN], o0[JIT_NLIVE], o1[JIT_NLIVE];
#pragma unroll
                for (uint32_t k = 0; k < JIT_NIN; ++k) { in0[k] = vin[j][k].x; in1[k] = vin[j][k].y; }
#pragma unroll
                for (uint32_t k = 0; k < JIT_NLIVE; ++k) { o0[k] = 0; o1[k] = 0; }
                bool a0 = row < P.n_rows, a1 = row + 1 < P.n_rows;
                uint32_t e0 = 0, e1 = 0;
                if (a0) jit_row_fixed(row, in0, a0, e0, o0);
                if (a1) jit_row_fixed(row + 1, in1, a1, e1, o1);
                al |= (a0 ? 1u : 0u) << (2 * j) | (a1 ? 2u : 0u) << (2 * j);
                ex |= (e0 ? 1u : 0u) << (2 * j) | (e1 ? 2u : 0u) << (2 * j);
                ec[2 * j] = e0;
                ec[2 * j + 1] = e1;
#pragma unroll
                for (uint32_t k = 0; k < JIT_NLIVE; ++k)
                    *reinterpret_cast<ulonglong2 *>(rb + k * SLOT_W + b * (TS * 8) + j * VV::SLAB) = make_ulonglong2(o0[k], o1[k]);
            }
            if (ex) {  // after the stores: the code takes the place of the (unwritten) row's slot 0
#pragma unroll
                for (uint32_t v = 0; v < 2 * J; ++v)
                    if ((ex >> v) & 1u) *code_at(b, VV::lrow(v >> 1, v & 1)) = ec[v];
            }
            alive[b] = al;
            excb[b] = ex;
        };
        if constexpr (JIT_NIN <= 2) {  // two sub-batches of input in registers: the next one is in flight while this one is evaluated
            ulonglong2 va[J][JIT_NIN], vb[J][JIT_NIN];
            jit_load_vec<J>(va, s_cols, base, P.n_rows, base + TS <= P.n_rows);
#pragma unroll
            for (uint32_t b = 0; b < B; b += 2) {
                jit_load_vec<J>(vb, s_cols, base + (uint64_t)(b + 1) * TS, P.n_rows, base + (uint64_t)(b + 2) * TS <= P.n_rows);
                eval(b, va);
                if (b + 2 < B) jit_load_vec<J>(va, s_cols, base + (uint64_t)(b + 2) * TS, P.n_rows, base + (uint64_t)(b + 3) * TS <= P.n_rows);
                eval(b + 1, vb);
            }
        } else {
#pragma unroll
            for (uint32_t b = 0; b < B; ++b) {
                ulonglong2 va[J][JIT_NIN];
                jit_load_vec<J>(va, s_cols, base + (uint64_t)b * TS, P.n_rows, base + (uint64_t)(b + 1) * TS <= P.n_rows);
                eval(b, va);
            }
        }

        // ---- counts per (sub-batch, slab, warp) group ----
        uint32_t any_exc = 0;
#pragma unroll
        for (uint32_t b = 0; b < B; ++b) any_exc |= excb[b];
        const bool warp_exc = __any_sync(0xFFFFFFFFu, any_exc != 0);
#pragma unroll
        for (uint32_t b = 0; b < B; ++b) {
#pragma unroll
            for (uint32_t j = 0; j < J; ++j) {
                const uint32_t ke = __ballot_sync(0xFFFFFFFFu, (alive[b] >> (2 * j)) & 1u), ko = __ballot_sync(0xFFFFFFFFu, (alive[b] >> (2 * j + 1)) & 1u);
                uint32_t cnt = __popc(ke) + __popc(ko);
                if (warp_exc) {
                    const uint32_t ee = __ballot_sync(0xFFFFFFFFu, (excb[b] >> (2 * j)) & 1u), eo = __ballot_sync(0xFFFFFFFFu, (excb[b] >> (2 * j + 1)) & 1u);
                    cnt |= (__popc(ee) + __popc(eo)) << 16;
                }
                if (lane == 0) s_cnt[b * 32 + j * 8 + warp] = cnt;
            }
        }
        __syncthreads();
        // every warp scans the B x 32 group counts (kept in the low half, raised in the high half: both <= T = 8192 < 2^16)
        uint32_t gex[B], run = 0;
#pragma unroll
        for (uint32_t b = 0; b < B; ++b) {
            uint32_t gi = s_cnt[b * 32 + lane];
            const uint32_t gmine = gi;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, gi, o);
                if (lane >= (uint32_t)o) gi += u;
            }
            gex[b] = run + gi - gmine;  // exclusive prefix of group (b, lane) inside the tile
            run += __shfl_sync(0xFFFFFFFFu, gi, 31);
        }
        const uint32_t n_keep = run & 0xFFFFu, n_exc = run >> 16;
        if (tid == 0)  // publish this tile's counts (tile 0: they are its inclusive prefix)
            st_cg_u64(P.tile_state + tile, ((uint64_t)(tile == 0 ? 2u : 1u) << 62) | ((uint64_t)n_keep << 31) | (uint64_t)n_exc);

        uint64_t pre_keep = 0, pre_exc = 0;
        vec_lookback(P, tile, n_keep, n_exc, s_scr, pre_keep, pre_exc);
        if (tid == 0 && tile == P.n_tiles - 1) {
            P.totals[0] = pre_keep + n_keep;
            P.totals[1] = pre_exc + n_exc;
        }

        // ---- write: every thread stores its own rows, straight from its column of the register file ----
        const bool exc_fit = pre_exc + n_exc <= P.cap_exc;
        if (n_exc && !exc_fit && tid == 0) atomicOr(&P.counters[1], 4u);
#pragma unroll
        for (uint32_t b = 0; b < B; ++b) {
#pragma unroll
            for (uint32_t j = 0; j < J; ++j) {
                const uint32_t a0 = (alive[b] >> (2 * j)) & 1u, a1 = (alive[b] >> (2 * j + 1)) & 1u;
                const uint32_t ke = __ballot_sync(0xFFFFFFFFu, a0), ko = __ballot_sync(0xFFFFFFFFu, a1);
                const uint32_t gpre = __shfl_sync(0xFFFFFFFFu, gex[b], j * 8 + warp);
                const uint32_t kk = (gpre & 0xFFFFu) + __popc(ke & lt) + __popc(ko & lt);  // kept rows of the tile before this thread's even row
                if (a0 | a1) {
                    const uint64_t at = pre_keep + kk;
                    for (uint32_t c = 0; c < P.n_out; ++c) {
                        const OutCol &oc = P.out[c];
                        uint64_t *od = oc.data;
                        __builtin_assume(__isGlobal(od));
                        const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(rb + oc.stage_off + b * (TS * 8) + j * VV::SLAB);
                        if (a0) od[at] = v.x;
                        if (a1) od[at + a0] = v.y;
                    }
                }
                if (n_exc && exc_fit) {  // uniform
                    const uint32_t x0 = (excb[b] >> (2 * j)) & 1u, x1 = (excb[b] >> (2 * j + 1)) & 1u;
                    const uint32_t ee = __ballot_sync(0xFFFFFFFFu, x0), eo = __ballot_sync(0xFFFFFFFFu, x1);
                    const uint32_t ek = (gpre >> 16) + __popc(ee & lt) + __popc(eo & lt);
                    for (uint32_t h = 0; h < 2; ++h) {
                        if (!(h ? x1 : x0)) continue;
                        const uint32_t lr = VV::lrow(j, h);
                        const uint32_t ke_ = ek + (h ? x0 : 0), kk_ = kk + (h ? a0 : 0);
                        tplx_exception_rec rec;
                        rec.row = (int64_t)(base + (uint64_t)b * TS + lr);
                        rec.row_no = P.first_row_no + (int64_t)(pre_keep + pre_exc + kk_ + ke_);  // rows written + exceptions so far (TransformTask.cc:764,885)
                        const uint32_t es = *code_at(b, lr);
                        rec.code = es & 0xFFFF;
                        rec.op_id = P.opids[es >> 16];
                        P.exc[pre_exc + ke_] = rec;
                    }
                }
            }
        }
        if (tid == 0) s_ctl[0] = atomicAdd(&P.counters[0], 1u);  // every thread read the old ticket before the counts barrier of this tile
    }
}
#endif  // K1w

#if defined(TPLX_JIT) && TPLX_JIT_KIND == 10
// ---- K1r: the specialised fixed-width row kernel that stages NOTHING: L2 is the staging buffer ----------------------------------------
// A tile of K1w goes through four phases: load + evaluate, counts, look-back (= waiting for the slowest load among the ~1000 tiles
// in flight: in-order retirement), stores. Rows sit in shared memory from their evaluation to their store, and shared memory
// bounds the rows in flight (132 SMs x 227 KB / 8 B = 3.8 M rows on H100): throughput = rows in flight / latency. Short of making DRAM
// latency deterministic, the way out is to hold rows in flight somewhere bigger: the 50 MB L2. K1r evaluates a tile TWICE:
//   pass 1: LDG.128 the inputs, run the row function for the row's FATE only (kept / filtered / raised: two bits per row in registers),
//           count, publish — nothing is staged;
//   pass 2: once the tile's offset is known, LDG.128 the same inputs again (read a few microseconds ago: L2 hits), run the row
//           function again and store the outputs of the kept rows straight from registers.
// DRAM traffic stays algorithmic (one read, one write), the second read costs L2 bandwidth and the second evaluation instructions — a
// trade for programs of a few operations (the planner picks K1r for those, K1w otherwise). No shared memory beyond the counts, so a
// CTA can keep TWO tiles in flight for the price of ten registers: the look-back of tile A (the wait for the slowest of its predecessors)
// is done after pass 1 of the CTA's next tile B has been issued and B's counts are published — the wait overlaps real work, and no
// ticket is ever held without its counts being produced as fast as the CTA can.
extern "C" __global__ void __launch_bounds__(NT, TPLX_JIT_MIN_CTAS) tplx_jit_kernel(const __grid_constant__ KParams P) {
    extern __shared__ __align__(16) uint8_t smem[];
    constexpr int J = 4, B = 2;
    using VV = VecVM<J>;
    constexpr uint32_t TS = VV::T, T = B * TS;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    ColIn *s_cols = reinterpret_cast<ColIn *>(smem + P.smem_cols_off);
    uint32_t *s_cnt = reinterpret_cast<uint32_t *>(smem + P.smem_misc_off);  // [B][32]: kept | raised << 16 per (sub-batch, slab, warp)
    uint64_t *s_scr = reinterpret_cast<uint64_t *>(s_cnt + B * 32);
    uint32_t *s_ctl = reinterpret_cast<uint32_t *>(s_scr + 4 * (NT / 32));

    for (uint32_t i = tid; i < P.n_in * (sizeof(ColIn) / 8); i += NT)
        reinterpret_cast<uint64_t *>(s_cols)[i] = reinterpret_cast<const uint64_t *>(P.in)[i];
    const uint32_t lt = (1u << lane) - 1u;

    struct Tile {            // what a thread keeps of a tile between its two passes
        uint32_t tile;       // ticket
        uint64_t alive, excm;  // bit b * 8 + v: row v of this thread in sub-batch b is kept / raised
        uint32_t gex[B];     // exclusive prefix (kept | raised << 16) of group (b, lane) inside the tile
        uint32_t n_keep, n_exc;
    };

    // pass 1 + counts + publication of tile t.tile (all threads; one barrier)
    auto first_pass = [&](Tile &t) {
        const uint64_t base = (uint64_t)t.tile * T;
        uint64_t alive = 0, excm = 0;
#pragma unroll
        for (uint32_t b = 0; b < B; ++b) {
            ulonglong2 vin[J][JIT_NIN];
            const uint64_t sb = base + (uint64_t)b * TS;
            jit_load_vec<J>(vin, s_cols, sb, P.n_rows, sb + TS <= P.n_rows);
#pragma unroll
            for (uint32_t j = 0; j < J; ++j) {
                const uint64_t row = sb + VV::lrow(j, 0);
                uint64_t in0[JIT_NIN], in1[JIT_NIN], o0[JIT_NLIVE], o1[JIT_NLIVE];
#pragma unroll
                for (uint32_t k = 0; k < JIT_NIN; ++k) { in0[k] = vin[j][k].x; in1[k] = vin[j][k].y; }
                bool a0 = row < P.n_rows, a1 = row + 1 < P.n_rows;
                uint32_t e0 = 0, e1 = 0;
                if (a0) jit_row_fixed(row, in0, a0, e0, o0);
                if (a1) jit_row_fixed(row + 1, in1, a1, e1, o1);
                alive |= (uint64_t)((a0 ? 1u : 0u) | (a1 ? 2u : 0u)) << (b * 8 + 2 * j);
                excm |= (uint64_t)((e0 ? 1u : 0u) | (e1 ? 2u : 0u)) << (b * 8 + 2 * j);
            }
        }
        const bool warp_exc = __any_sync(0xFFFFFFFFu, excm != 0);
#pragma unroll
        for (uint32_t b = 0; b < B; ++b) {
#pragma unroll
            for (uint32_t j = 0; j < J; ++j) {
                const uint32_t sh = b * 8 + 2 * j;
                const uint32_t ke = __ballot_sync(0xFFFFFFFFu, (alive >> sh) & 1u), ko = __ballot_sync(0xFFFFFFFFu, (alive >> (sh + 1)) & 1u);
                uint32_t cnt = __popc(ke) + __popc(ko);
                if (warp_exc) {
                    const uint32_t ee = __ballot_sync(0xFFFFFFFFu, (excm >> sh) & 1u), eo = __ballot_sync(0xFFFFFFFFu, (excm >> (sh + 1)) & 1u);
                    cnt |= (__popc(ee) + __popc(eo)) << 16;
                }
                if (lane == 0) s_cnt[b * 32 + j * 8 + warp] = cnt;
            }
        }
        __syncthreads();
        uint32_t run = 0;  // kept in the low half, raised in the high half: both <= T = 4096 < 2^16
#pragma unroll
        for (uint32_t b = 0; b < B; ++b) {
            uint32_t gi = s_cnt[b * 32 + lane];
            const uint32_t gmine = gi;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, gi, o);
                if (lane >= (uint32_t)o) gi += u;
            }
            t.gex[b] = run + gi - gmine;
            run += __shfl_sync(0xFFFFFFFFu, gi, 31);
        }
        t.alive = alive;
        t.excm = excm;
        t.n_keep = run & 0xFFFFu;
        t.n_exc = run >> 16;
        if (tid == 0)
            st_cg_u64(P.tile_state + t.tile, ((uint64_t)(t.tile == 0 ? 2u : 1u) << 62) | ((uint64_t)t.n_keep << 31) | (uint64_t)t.n_exc);
    };

    // look-back + pass 2 of a tile whose counts were published earlier
    auto second_pass = [&](const Tile &t) {
        const uint64_t base = (uint64_t)t.tile * T;
        uint64_t pre_keep = 0, pre_exc = 0;
        vec_lookback(P, t.tile, t.n_keep, t.n_exc, s_scr, pre_keep, pre_exc);
        if (tid == 0 && t.tile == P.n_tiles - 1) {
            P.totals[0] = pre_keep + t.n_keep;
            P.totals[1] = pre_exc + t.n_exc;
        }
        const bool exc_fit = pre_exc + t.n_exc <= P.cap_exc;
        if (t.n_exc && !exc_fit && tid == 0) atomicOr(&P.counters[1], 4u);
        if (!(t.n_keep || (t.n_exc && exc_fit))) return;  // uniform
#pragma unroll
        for (uint32_t b = 0; b < B; ++b) {
            if (!__any_sync(0xFFFFFFFFu, ((t.alive | t.excm) >> (b * 8)) & 0xFFu)) continue;  // nothing of this warp's rows in the sub-batch
            ulonglong2 vin[J][JIT_NIN];
            const uint64_t sb = base + (uint64_t)b * TS;
            jit_load_vec<J>(vin, s_cols, sb, P.n_rows, sb + TS <= P.n_rows);
#pragma unroll
            for (uint32_t j = 0; j < J; ++j) {
                const uint32_t sh = b * 8 + 2 * j;
                const uint32_t a0 = (uint32_t)(t.alive >> sh) & 1u, a1 = (uint32_t)(t.alive >> (sh + 1)) & 1u;
                const uint32_t x0 = (uint32_t)(t.excm >> sh) & 1u, x1 = (uint32_t)(t.excm >> (sh + 1)) & 1u;
                const uint64_t row = sb + VV::lrow(j, 0);
                uint64_t in0[JIT_NIN], in1[JIT_NIN], o0[JIT_NLIVE], o1[JIT_NLIVE];
#pragma unroll
                for (uint32_t k = 0; k < JIT_NIN; ++k) { in0[k] = vin[j][k].x; in1[k] = vin[j][k].y; }
#pragma unroll
                for (uint32_t k = 0; k < JIT_NLIVE; ++k) { o0[k] = 0; o1[k] = 0; }
                bool r0 = true, r1 = true;
                uint32_t e0 = 0, e1 = 0;
                if (a0 | x0) jit_row_fixed(row, in0, r0, e0, o0);      // same inputs, same function: same fate as in pass 1
                if (a1 | x1) jit_row_fixed(row + 1, in1, r1, e1, o1);
                const uint32_t ke = __ballot_sync(0xFFFFFFFFu, a0), ko = __ballot_sync(0xFFFFFFFFu, a1);
                const uint32_t gpre = __shfl_sync(0xFFFFFFFFu, t.gex[b], j * 8 + warp);
                const uint32_t kk = (gpre & 0xFFFFu) + __popc(ke & lt) + __popc(ko & lt);
                if (a0 | a1) {
                    const uint64_t at = pre_keep + kk;
#pragma unroll
                    for (uint32_t c = 0; c < JIT_NOUT; ++c) {
                        if (c >= P.n_out) break;
                        uint64_t *od = P.out[c].data;
                        __builtin_assume(__isGlobal(od));
                        if (a0) od[at] = o0[jit_outslot(c)];
                        if (a1) od[at + a0] = o1[jit_outslot(c)];
                    }
                }
                if (t.n_exc && exc_fit) {  // uniform
                    const uint32_t ee = __ballot_sync(0xFFFFFFFFu, x0), eo = __ballot_sync(0xFFFFFFFFu, x1);
                    const uint32_t ek = (gpre >> 16) + __popc(ee & lt) + __popc(eo & lt);
                    for (uint32_t h = 0; h < 2; ++h) {
                        if (!(h ? x1 : x0)) continue;
                        const uint32_t ke_ = ek + (h ? x0 : 0), kk_ = kk + (h ? a0 : 0);
                        tplx_exception_rec rec;
                        rec.row = (int64_t)(sb + VV::lrow(j, h));
                        rec.row_no = P.first_row_no + (int64_t)(pre_keep + pre_exc + kk_ + ke_);  // rows written + exceptions so far (TransformTask.cc:764,885)
                        const uint32_t es = h ? e1 : e0;
                        rec.code = es & 0xFFFF;
                        rec.op_id = P.opids[es >> 16];
                        P.exc[pre_exc + ke_] = rec;
                    }
                }
            }
        }
    };

    // Two tiles in flight per CTA: pass 1 of the new ticket first (its counts are what every successor waits for), then the
    // look-back + pass 2 of the previous one.
    Tile cur, prev;
    bool have_prev = false;
    if (tid == 0) s_ctl[0] = atomicAdd(&P.counters[0], 1u);
    while (true) {
        __syncthreads();  // the ticket is visible; s_cnt and the look-back scratch are free again
        cur.tile = s_ctl[0];
        const bool have = cur.tile < P.n_tiles;  // uniform
        if (have) first_pass(cur);
        if (have_prev) second_pass(prev);
        if (!have) break;
        prev = cur;
        have_prev = true;
        if (tid == 0) s_ctl[0] = atomicAdd(&P.counters[0], 1u);  // every thread has read the old ticket (barrier of first_pass)
    }
}
#endif  // K1r

#if !defined(TPLX_JIT) || TPLX_JIT_KIND == 2 || TPLX_JIT_KIND == 3
#ifdef TPLX_JIT
extern "C" __global__ void __launch_bounds__(NT, TPLX_JIT_MIN_CTAS) tplx_jit_kernel(const __grid_constant__ KParams P) {
    constexpr int J = TPLX_JIT_KIND == 3 ? 2 : 4;
#else
template <int J>
__global__ void __launch_bounds__(NT, 4) stage_rows_vec_kernel(const __grid_constant__ KParams P) {  // parameters in the constant bank
#endif
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr uint32_t T = VecVM<J>::T, G = 8 * J;  // G = (slab, warp) groups per tile (<= 32)
    static_assert(G <= 32, "one scan lane per (slab, warp) group");

    VInstr *s_prog = reinterpret_cast<VInstr *>(smem);
    ColIn *s_cols = reinterpret_cast<ColIn *>(smem + P.smem_cols_off);
    uint8_t *s_regs = smem + P.smem_regs_off;
    uint32_t *s_cnt = reinterpret_cast<uint32_t *>(smem + P.smem_misc_off);
    uint32_t *exc_stage = s_cnt + 32;
    uint64_t *s_scr = reinterpret_cast<uint64_t *>(exc_stage + T);  // look-back scratch: 2 words per warp, double-buffered
    uint32_t *s_ctl = reinterpret_cast<uint32_t *>(s_scr + 4 * (NT / 32));  // [0] ticket

    for (uint32_t i = tid; i < P.n_instr * (sizeof(VInstr) / 16); i += NT)
        reinterpret_cast<uint4 *>(s_prog)[i] = reinterpret_cast<const uint4 *>(P.prog)[i];
    for (uint32_t i = tid; i < P.n_in * (sizeof(ColIn) / 8); i += NT)
        reinterpret_cast<uint64_t *>(s_cols)[i] = reinterpret_cast<const uint64_t *>(P.in)[i];
    uint8_t *rb = s_regs + tid * 16;
    const uint32_t lt = (1u << lane) - 1u;

    // Tickets are taken when the tile starts, not ahead of time: a ticket held while its owner still works on the previous tile
    // stalls the look-back of every later tile (so does loading the next tile's input under the look-back of this one: both were slower
    // on C1). Thread 0 takes the next ticket when IT has finished the
    // tile (its atomic overlaps the other warps' stores) and one barrier at the top of the loop publishes it.
    if (tid == 0) s_ctl[0] = atomicAdd(&P.counters[0], 1u);
    while (true) {
        __syncthreads();  // the ticket is visible; s_cnt and the look-back scratch of the previous tile are no longer read
        const uint32_t tile = s_ctl[0];
        if (tile >= P.n_tiles) break;
        const uint64_t base = (uint64_t)tile * T;
        const bool full = base + T <= P.n_rows;  // uniform

        typename VecVM<J>::State st;
        st.exc = 0;
        if (full) st.alive = (1u << (2 * J)) - 1u;  // every row starts alive
        else {
            st.alive = 0;
#pragma unroll
            for (uint32_t v = 0; v < 2 * J; ++v)
                if (base + VecVM<J>::lrow(v >> 1, v & 1) < P.n_rows) st.alive |= 1u << v;
        }
#if defined(TPLX_JIT)
        {
            ulonglong2 vin[J][JIT_NIN];
            jit_load_vec<J>(vin, s_cols, base, P.n_rows, full);
            jit_eval_vec<J>(vin, rb, base, st, exc_stage);
        }
#else
        VecVM<J>::run(s_prog, P.n_instr, smem, rb, s_cols, base, P.n_rows, full, st, exc_stage);
#endif

        // ---- counts per (slab, warp) group ----
        const bool warp_exc = __any_sync(0xFFFFFFFFu, st.exc != 0);
#pragma unroll
        for (uint32_t j = 0; j < J; ++j) {
            const uint32_t ke = __ballot_sync(0xFFFFFFFFu, (st.alive >> (2 * j)) & 1u), ko = __ballot_sync(0xFFFFFFFFu, (st.alive >> (2 * j + 1)) & 1u);
            uint32_t cnt = __popc(ke) + __popc(ko);
            if (warp_exc) {
                const uint32_t ee = __ballot_sync(0xFFFFFFFFu, (st.exc >> (2 * j)) & 1u), eo = __ballot_sync(0xFFFFFFFFu, (st.exc >> (2 * j + 1)) & 1u);
                cnt |= (__popc(ee) + __popc(eo)) << 16;
            }
            if (lane == 0) s_cnt[j * 8 + warp] = cnt;
        }
        __syncthreads();
        // every warp scans the G group counts (kept in the low half, raised in the high half: both <= T = 2048)
        uint32_t gi = lane < G ? s_cnt[lane] : 0;
        const uint32_t gmine = gi;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, gi, o);
            if (lane >= (uint32_t)o) gi += u;
        }
        const uint32_t gtot = __shfl_sync(0xFFFFFFFFu, gi, 31);
        const uint32_t gex = gi - gmine;  // exclusive prefix of group `lane`
        const uint32_t n_keep = gtot & 0xFFFFu, n_exc = gtot >> 16;
        if (tid == 0)  // publish this tile's counts (tile 0: they are its inclusive prefix)
            st_cg_u64(P.tile_state + tile, ((uint64_t)(tile == 0 ? 2u : 1u) << 62) | ((uint64_t)n_keep << 31) | (uint64_t)n_exc);

        // ---- look-back: 256 predecessors per round ----
        uint64_t pre_keep = 0, pre_exc = 0;
        vec_lookback(P, tile, n_keep, n_exc, s_scr, pre_keep, pre_exc);
        if (tid == 0 && tile == P.n_tiles - 1) {
            P.totals[0] = pre_keep + n_keep;
            P.totals[1] = pre_exc + n_exc;
        }

        // ---- write: every thread stores its own rows, straight from its column of the register file ----
        const bool exc_fit = pre_exc + n_exc <= P.cap_exc;
        if (n_exc && !exc_fit && tid == 0) atomicOr(&P.counters[1], 4u);
#pragma unroll
        for (uint32_t j = 0; j < J; ++j) {
            const uint32_t a0 = (st.alive >> (2 * j)) & 1u, a1 = (st.alive >> (2 * j + 1)) & 1u;
            const uint32_t ke = __ballot_sync(0xFFFFFFFFu, a0), ko = __ballot_sync(0xFFFFFFFFu, a1);
            const uint32_t gpre = __shfl_sync(0xFFFFFFFFu, gex, j * 8 + warp);
            const uint32_t kk = (gpre & 0xFFFFu) + __popc(ke & lt) + __popc(ko & lt);  // kept rows of the tile before this thread's even row
            if (a0 | a1) {
                const uint64_t at = pre_keep + kk;
                for (uint32_t c = 0; c < P.n_out; ++c) {
                    const OutCol &oc = P.out[c];
                    uint64_t *od = oc.data;
                    __builtin_assume(__isGlobal(od));
                    const ulonglong2 v = VecVM<J>::ld2(rb, oc.stage_off, j);
                    if (a0) od[at] = v.x;
                    if (a1) od[at + a0] = v.y;
                }
            }
            if (n_exc && exc_fit) {  // uniform
                const uint32_t x0 = (st.exc >> (2 * j)) & 1u, x1 = (st.exc >> (2 * j + 1)) & 1u;
                const uint32_t ee = __ballot_sync(0xFFFFFFFFu, x0), eo = __ballot_sync(0xFFFFFFFFu, x1);
                const uint32_t ek = (gpre >> 16) + __popc(ee & lt) + __popc(eo & lt);
                for (uint32_t b = 0; b < 2; ++b) {
                    if (!(b ? x1 : x0)) continue;
                    const uint32_t lr = VecVM<J>::lrow(j, b);
                    const uint32_t ke_ = ek + (b ? x0 : 0), kk_ = kk + (b ? a0 : 0);
                    tplx_exception_rec rec;
                    rec.row = (int64_t)(base + lr);
                    rec.row_no = P.first_row_no + (int64_t)(pre_keep + pre_exc + kk_ + ke_);  // rows written + exceptions so far (TransformTask.cc:764,885)
                    const uint32_t es = exc_stage[lr];
                    rec.code = es & 0xFFFF;
                    rec.op_id = P.opids[es >> 16];
                    P.exc[pre_exc + ke_] = rec;
                }
            }
        }
        if (tid == 0) s_ctl[0] = atomicAdd(&P.counters[0], 1u);  // every thread read the old ticket before the counts barrier of this tile
    }
}
#endif  // K1v

}  // namespace tplx
