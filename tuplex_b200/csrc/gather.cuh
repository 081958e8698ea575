// gather.cuh — device columns built from selected rows of other columns: the late materialisation below, and the gather by row
// selector of join and merge outputs at the end of the file.
//
// Late materialisation of "late" columns for the rows a prefilter stage let through.
// When the inputs of tplx_gpu_stage_run_host lie in page-locked host memory, only the columns the prefilter
// reads are copied to HBM up front. The remaining columns are needed for the surviving rows only: these kernels
// read exactly those rows through the mapped host address (many independent, coalesced reads in flight, so the
// transfer is PCIe-bandwidth bound rather than latency bound) and build compact device columns indexed by the
// position in the survivor list. The dense launch then addresses them with the work index instead of the row.
// (The reference has no counterpart: it always deserialises whole rows, TuplexSourceTaskBuilder.cc:184-189.)
#pragma once
#include <stdint.h>
#include "vm.cuh"
#include "csvops.cuh"

namespace tplx {

constexpr uint64_t COL_COMPACT = 0x100;  // ColIn.type flag: column is indexed by work position, not by input row

struct GatherCols {
    uint32_t n_cols;
    uint32_t pad;
    uint8_t type[TPLX_MAX_COLS];
    const void *src_data[TPLX_MAX_COLS];
    const uint32_t *src_off[TPLX_MAX_COLS];
    uint64_t *dst_data[TPLX_MAX_COLS];   // fixed width
    uint32_t *dst_off[TPLX_MAX_COLS];    // strings: n+1 offsets
    uint8_t *dst_bytes[TPLX_MAX_COLS];
    uint64_t *lens[TPLX_MAX_COLS];       // strings: length per survivor (then exclusive scan), n+1 entries
    uint32_t *srcpos[TPLX_MAX_COLS];     // strings: source byte offset per survivor
    // lazy columns of a CSV block (K6): src_data = the CSV text, src_ref[c][row] = start | raw_len << 32 | escaped << 63
    const uint64_t *src_ref[TPLX_MAX_COLS];
    uint8_t quote;
};

// one thread per (survivor, column): fixed-width values and string lengths
__global__ void gather_pass1(const uint64_t *__restrict__ rowlist, uint64_t n, const GatherCols *__restrict__ G) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t row = rowlist[i];
    for (uint32_t c = 0; c < G->n_cols; ++c) {
        if (G->type[c] == TPLX_T_STR && G->src_ref[c]) {
            const uint64_t info = G->src_ref[c][row];
            const uint32_t b = (uint32_t)info, raw = (uint32_t)(info >> 32) & 0x7FFFFFFFu;
            G->lens[c][i] = (info >> 63) ? csv_dequoted_len(reinterpret_cast<const uint8_t *>(G->src_data[c]), b, b + raw, G->quote) : raw;
            G->srcpos[c][i] = b;
        } else if (G->type[c] == TPLX_T_STR) {
            const uint2 o = make_uint2(G->src_off[c][row], G->src_off[c][row + 1]);
            G->lens[c][i] = o.y - o.x;
            G->srcpos[c][i] = o.x;
        } else {
            G->dst_data[c][i] = reinterpret_cast<const uint64_t *>(G->src_data[c])[row];
        }
    }
}

// one warp per survivor: copy the bytes of every string column (lanes read consecutive bytes -> coalesced)
__global__ void gather_pass2(uint64_t n, const GatherCols *__restrict__ G, const uint64_t *__restrict__ rowlist) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (i > n) return;
    for (uint32_t c = 0; c < G->n_cols; ++c) {
        if (G->type[c] != TPLX_T_STR) continue;
        const uint64_t d0 = G->lens[c][i];  // exclusive scan: destination offset (entry n = total)
        if (lane == 0) G->dst_off[c][i] = (uint32_t)d0;
        if (i == n) continue;
        const uint32_t len = (uint32_t)(G->lens[c][i + 1] - d0);
        const uint8_t *src = reinterpret_cast<const uint8_t *>(G->src_data[c]) + G->srcpos[c][i];
        uint8_t *dst = G->dst_bytes[c] + d0;
        if (G->src_ref[c] && (G->src_ref[c][rowlist[i]] >> 63)) {  // cell with doubled quotes: dequoted by one lane
            if (lane == 0) {
                const uint32_t raw = (uint32_t)(G->src_ref[c][rowlist[i]] >> 32) & 0x7FFFFFFFu;
                csv_dequote(src, 0, raw, G->quote, dst, len);
            }
            continue;
        }
        for (uint32_t k = lane; k < len; k += 32) dst[k] = src[k];
    }
}

// ---- gather by row selector: output columns built from rows of up to two device columns (K8 join outputs, K9 merge) ----------
// One u32 selector per output row. SEL_NONE: no source row (value 0, length 0, validity bit clear). Otherwise the row is
// s & ~b_bit of source B when s & b_bit, else of source A. A source without a bitmap gives set bits. Sources are read with __ldg:
// a pointer picked from a struct is not known to be global memory, and a plain load would not take the read-only path.
constexpr uint32_t SEL_NONE = 0xFFFFFFFFu;
constexpr uint32_t SEL_NT = 256;
constexpr uint32_t SEL_STR_LANES = 8;  // lanes that copy one output string

struct SelSrc {
    const void *data;         // 8-byte values, or string bytes
    const uint32_t *offsets;  // strings: n + 1 offsets
    const uint32_t *valid;    // validity bitmap, or nullptr
};

__device__ __forceinline__ SelSrc sel_src(uint32_t s, uint32_t b_bit, const SelSrc &a, const SelSrc &b, uint32_t *row) {
    *row = s & ~b_bit;
    return (s & b_bit) ? b : a;
}

__global__ void __launch_bounds__(SEL_NT) sel_gather_fixed_kernel(SelSrc a, SelSrc b, uint32_t b_bit, const uint32_t *__restrict__ sel, uint64_t n,
                                                                   uint64_t *__restrict__ dst) {
    const uint64_t i = (uint64_t)blockIdx.x * SEL_NT + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = sel[i];
    if (s == SEL_NONE) { dst[i] = 0; return; }
    uint32_t r;
    const SelSrc src = sel_src(s, b_bit, a, b, &r);
    dst[i] = __ldg(static_cast<const uint64_t *>(src.data) + r);
}

// one validity word per warp
__global__ void __launch_bounds__(SEL_NT) sel_gather_valid_kernel(SelSrc a, SelSrc b, uint32_t b_bit, const uint32_t *__restrict__ sel, uint64_t n,
                                                                   uint32_t *__restrict__ dst_words) {
    const uint64_t i = (uint64_t)blockIdx.x * SEL_NT + threadIdx.x;
    bool ok = false;
    if (i < n) {
        const uint32_t s = sel[i];
        if (s != SEL_NONE) {
            uint32_t r;
            const uint32_t *v = sel_src(s, b_bit, a, b, &r).valid;
            ok = !v || ((__ldg(v + (r >> 5)) >> (r & 31)) & 1u);
        }
    }
    const uint32_t w = __ballot_sync(0xFFFFFFFFu, ok);
    if ((threadIdx.x & 31) == 0 && (i >> 5) < ((n + 31) >> 5)) dst_words[i >> 5] = w;
}

// strings: lengths (then an exclusive scan in place), then the bytes
__global__ void __launch_bounds__(SEL_NT) sel_str_len_kernel(SelSrc a, SelSrc b, uint32_t b_bit, const uint32_t *__restrict__ sel, uint64_t n,
                                                              uint64_t *__restrict__ lens) {
    const uint64_t i = (uint64_t)blockIdx.x * SEL_NT + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = sel[i];
    if (s == SEL_NONE) { lens[i] = 0; return; }
    uint32_t r;
    const uint32_t *o = sel_src(s, b_bit, a, b, &r).offsets;
    lens[i] = __ldg(o + r + 1) - __ldg(o + r);
}

__global__ void __launch_bounds__(SEL_NT) sel_str_copy_kernel(SelSrc a, SelSrc b, uint32_t b_bit, const uint32_t *__restrict__ sel, uint64_t n,
                                                               const uint64_t *__restrict__ pos, uint32_t *__restrict__ dst_off, uint8_t *__restrict__ dst) {
    // SEL_STR_LANES lanes per output row: the strings of these paths are short (codes, names: 8 B in the bench's join table), so a
    // whole warp per row would leave most lanes idle; 8 lanes keep one byte per lane and row in flight
    const uint64_t t = (uint64_t)blockIdx.x * SEL_NT + threadIdx.x;
    const uint64_t i = t / SEL_STR_LANES;
    const uint32_t sub = (uint32_t)(t % SEL_STR_LANES);
    if (i > n) return;
    const uint64_t d0 = pos[i];
    if (sub == 0) dst_off[i] = (uint32_t)d0;  // entry n = total
    if (i == n) return;
    const uint32_t s = sel[i];
    if (s == SEL_NONE) return;
    uint32_t r;
    const SelSrc src = sel_src(s, b_bit, a, b, &r);
    const uint8_t *bytes = static_cast<const uint8_t *>(src.data);
    const uint32_t s0 = __ldg(src.offsets + r), len = __ldg(src.offsets + r + 1) - s0;
    for (uint32_t k = sub; k < len; k += SEL_STR_LANES) dst[d0 + k] = __ldg(bytes + s0 + k);
}

// survivor list (mask_expand_kernel writes u64 row numbers) -> u32 selectors of the kernels above (tplx_gpu_block_select). The
// gathers take 32-bit selectors because the merge and join mark the second source in the top bit; mask.cuh's list stays 64-bit
// for the stage kernels that share it.
__global__ void __launch_bounds__(SEL_NT) sel_from_rows_kernel(const uint64_t *__restrict__ rows, uint64_t n, uint32_t *__restrict__ sel) {
    const uint64_t i = (uint64_t)blockIdx.x * SEL_NT + threadIdx.x;
    if (i < n) sel[i] = (uint32_t)rows[i];
}

}  // namespace tplx
