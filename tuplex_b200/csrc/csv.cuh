// csv.cuh — K6: CSV bytes -> column block, on the device.
//
// Replaces the reference's host CSV source for a TransformStage: CSVReader::read + csvmonkey row splitting
// (tuplex/core/src/physical/CSVReader.cc:388-634, core/include/physical/csvmonkey.h:523-672) and the cell decoding the
// stage function starts with (decodeCells, codegen/src/FlattenedTuple.cc:1215-1330). Semantics live in csvops.cuh.
//
// The reference parses sequentially; here rows are found in parallel and then checked:
//   1. csv_tile_states   per 64-byte span: quote parity + row ends counted for both possible start states; a
//                        block scan composes spans into one state per 16 KB tile
//   2. csv_scan_tiles    one block: exclusive scan of the tile states (start parity, rows before) per tile
//   3. csv_row_ends      same walk with the now known start state: position of every row-ending newline
//   4. csv_parse_rows    one thread per row runs the reference's exact row machine (csvops.cuh), decodes the selected
//                        cells, and VERIFIES that the machine ends on the newline step 3 predicted. Quote parity is a
//                        speculation that is exact for well-formed CSV; if any row disagrees (stray quotes) or the file
//                        ends inside quotes, the host reruns row finding with csv_rows_sequential (one thread, the
//                        exact machine) — still on the device, no CPU fallback.
//   5. scans + csv_compact + csv_copy_strings   good rows are compacted into dense columns (strings dequoted and
//                        packed); rows that do not fit the normal case (cell count, null in a non-Option column,
//                        conversion error) become exception entries for the interpreter path, like
//                        BADPARSE_STRING_INPUT rows in the reference (CSVReader.cc:470-520,583-600).
//   6. csv_pack_valid    Option[T] columns only: a null cell there is None (step 4 records it in the row's null mask),
//                        and the validity words of the block follow from the masks in block row order.
// HBM-bound byte work: coalesced 16-byte loads, no tensor cores. Algorithmic traffic per input byte: read 3x (steps
// 1,3,4) + string payload read+written once.
#pragma once
#include <stdint.h>
#include "csvops.cuh"
#include "../../include/tplx_gpu.h"

namespace tplx {

constexpr int CSV_NT = 256;
constexpr uint32_t CSV_TILE = CSV_NT * CSV_SPAN;  // 16 KB per CTA

__device__ __forceinline__ CsvState csv_shfl_up(const CsvState &s, int o) {
    CsvState r;
    r.par = __shfl_up_sync(0xFFFFFFFFu, s.par, o);
    r.c0 = __shfl_up_sync(0xFFFFFFFFu, s.c0, o);
    r.c1 = __shfl_up_sync(0xFFFFFFFFu, s.c1, o);
    return r;
}

// exclusive block scan (CSV_NT threads) of span states; returns this thread's prefix and the block total
__device__ __forceinline__ CsvState csv_block_scan(const CsvState &mine, CsvState *total) {
    __shared__ CsvState warp_tot[CSV_NT / 32];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    CsvState inc = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        CsvState a = csv_shfl_up(inc, o);
        if (lane >= (uint32_t)o) inc = csv_compose(a, inc);
    }
    if (lane == 31) warp_tot[wid] = inc;
    CsvState ex = csv_shfl_up(inc, 1);
    if (lane == 0) ex = CsvState{0, 0, 0};
    __syncthreads();
    CsvState pre{0, 0, 0};
    for (uint32_t w = 0; w < wid; ++w) pre = csv_compose(pre, warp_tot[w]);
    if (total) {
        CsvState t = pre;
        for (uint32_t w = wid; w < CSV_NT / 32; ++w) t = csv_compose(t, warp_tot[w]);
        *total = t;
    }
    __syncthreads();
    return csv_compose(pre, ex);
}

// span state packed for step 3: parity | c0 << 8 | c1 << 16 (counts <= 64)
__global__ void __launch_bounds__(CSV_NT) csv_tile_states(const uint8_t *__restrict__ buf, uint8_t quote, CsvState *__restrict__ tiles,
                                                          uint32_t *__restrict__ span_state) {
    const uint64_t start = (uint64_t)blockIdx.x * CSV_TILE + (uint64_t)threadIdx.x * CSV_SPAN;
    CsvState s = csv_walk_span(buf, start, quote, 1u << 31, [](uint64_t) {});
    span_state[(size_t)blockIdx.x * CSV_NT + threadIdx.x] = s.par | (s.c0 << 8) | (s.c1 << 16);
    CsvState tot;
    csv_block_scan(s, &tot);
    if (threadIdx.x == 0) tiles[blockIdx.x] = tot;
}

// one block of 1024 threads; tile_start[t] = {parity, rows} before tile t, totals = {final parity, row count}
__global__ void __launch_bounds__(1024) csv_scan_tiles(const CsvState *__restrict__ tiles, uint32_t n_tiles, uint2 *__restrict__ tile_start,
                                                       uint32_t *__restrict__ totals) {
    __shared__ CsvState warp_tot[32];
    const uint32_t per = (n_tiles + 1023) / 1024;
    const uint32_t t0 = threadIdx.x * per, t1 = min(n_tiles, t0 + per);
    CsvState agg{0, 0, 0};
    for (uint32_t t = t0; t < t1; ++t) agg = csv_compose(agg, tiles[t]);
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    CsvState inc = agg;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        CsvState a = csv_shfl_up(inc, o);
        if (lane >= (uint32_t)o) inc = csv_compose(a, inc);
    }
    if (lane == 31) warp_tot[wid] = inc;
    CsvState ex = csv_shfl_up(inc, 1);
    if (lane == 0) ex = CsvState{0, 0, 0};
    __syncthreads();
    CsvState pre{0, 0, 0};
    for (uint32_t w = 0; w < wid; ++w) pre = csv_compose(pre, warp_tot[w]);
    pre = csv_compose(pre, ex);
    uint32_t par = pre.par, rows = pre.c0;  // the file starts outside quotes
    for (uint32_t t = t0; t < t1; ++t) {
        tile_start[t] = make_uint2(par, rows);
        const CsvState s = tiles[t];
        rows += par ? s.c1 : s.c0;
        par ^= s.par;
    }
    if (threadIdx.x == 1023) {
        totals[0] = par;
        totals[1] = rows;
    }
}

__global__ void __launch_bounds__(CSV_NT) csv_row_ends(const uint8_t *__restrict__ buf, uint8_t quote, const uint2 *__restrict__ tile_start,
                                                       const uint32_t *__restrict__ span_state, uint32_t *__restrict__ row_end) {
    const uint64_t start = (uint64_t)blockIdx.x * CSV_TILE + (uint64_t)threadIdx.x * CSV_SPAN;
    const uint32_t packed = span_state[(size_t)blockIdx.x * CSV_NT + threadIdx.x];  // step 1's walk, not repeated
    CsvState s{packed & 1u, (packed >> 8) & 0xFFu, (packed >> 16) & 0xFFu};
    const CsvState pre = csv_block_scan(s, nullptr);
    const uint2 ts = tile_start[blockIdx.x];
    const uint32_t par0 = ts.x ^ pre.par;
    uint32_t row = ts.y + (ts.x ? pre.c1 : pre.c0);
    if ((s.c0 | s.c1) == 0) return;
    csv_walk_span(buf, start, quote, par0, [&](uint64_t pos) { row_end[row++] = (uint32_t)pos; });
}

// exact, sequential row finding (repair path for irregular quoting)
__global__ void csv_rows_sequential(const uint8_t *__restrict__ buf, uint32_t n, uint8_t delim, uint8_t quote, uint32_t *__restrict__ row_end,
                                    uint32_t *__restrict__ totals) {
    if (threadIdx.x || blockIdx.x) return;
    totals[0] = 0;
    totals[1] = csv_find_rows_sequential(buf, n, delim, quote, row_end);
}

__global__ void __launch_bounds__(CSV_NT) csv_parse_rows(const CsvParseParams P) {
    const uint32_t i = blockIdx.x * CSV_NT + threadIdx.x;
    if (i < P.nd) csv_parse_one_row(P, i);
}

struct CsvCompactParams {
    uint32_t nd, r0, n_out, n_str;
    uint8_t quote;
    uint8_t out_types[TPLX_MAX_COLS];
    int8_t strk[TPLX_MAX_COLS];
    const uint64_t *tmp[TPLX_MAX_COLS];
    const uint64_t *lens;  // scanned: exclusive offsets, [k][nd] = total
    const uint64_t *good;  // scanned: output position, [nd] = n_good
    const uint32_t *code;
    const uint32_t *row_end;
    const uint8_t *buf;
    uint64_t *data[TPLX_MAX_COLS];
    uint32_t *offsets[TPLX_MAX_COLS];
    uint8_t *bytes[TPLX_MAX_COLS];
    uint64_t *refs[TPLX_MAX_COLS];  // lazy string columns (strk < 0): the cell reference of every good row
    uint32_t *rowmap;
    tplx_csv_bad_row *bad;
};

__global__ void __launch_bounds__(CSV_NT) csv_compact(const CsvCompactParams P) {
    const uint32_t i = blockIdx.x * CSV_NT + threadIdx.x;
    if (i >= P.nd) return;
    const uint64_t pos = P.good[i];
    const uint32_t code = P.code[i];
    if (code) {
        const uint32_t r = P.r0 + i;
        uint32_t s = r == 0 ? 0u : P.row_end[r - 1] + 1;
        while (csv_is_nl(P.buf[s])) ++s;
        tplx_csv_bad_row b;
        b.row = i;
        b.code = code;
        b.line_start = s;
        b.line_end = P.row_end[r];
        P.bad[i - pos] = b;
        return;
    }
    P.rowmap[pos] = i;
    for (uint32_t c = 0; c < P.n_out; ++c) {
        if (P.out_types[c] == TPLX_T_STR && P.strk[c] < 0)
            P.refs[c][pos] = P.tmp[c][i];
        else if (P.out_types[c] == TPLX_T_STR)
            P.offsets[c][pos] = (uint32_t)P.lens[(size_t)P.strk[c] * (P.nd + 1) + i];
        else
            P.data[c][pos] = P.tmp[c][i];
    }
    if (pos + 1 == P.good[P.nd])  // last good row also writes the closing offsets
        for (uint32_t c = 0; c < P.n_out; ++c)
            if (P.out_types[c] == TPLX_T_STR && P.strk[c] >= 0) P.offsets[c][pos + 1] = (uint32_t)P.lens[(size_t)P.strk[c] * (P.nd + 1) + P.nd];
}

// One warp per 32 consecutive rows; lane i first loads row i's cell info and output offset (coalesced), then the warp
// copies four cells at a time: 8 lanes per cell, consecutive lanes on consecutive bytes (rows are consecutive in the
// destination, so the four groups write one contiguous region). Cells with doubled quotes (rare) are dequoted by the
// first lane of their group.
__global__ void __launch_bounds__(CSV_NT) csv_copy_strings(const CsvCompactParams P) {
    const uint32_t g = (blockIdx.x * CSV_NT + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t r_first = g * 32;
    if (r_first >= P.nd) return;
    const uint32_t i = r_first + lane;
    const bool mine = i < P.nd && P.code[i] == 0;
    const uint32_t sub = lane >> 3, k0 = lane & 7;
    for (uint32_t c = 0; c < P.n_out; ++c) {
        if (P.out_types[c] != TPLX_T_STR || P.strk[c] < 0) continue;
        const uint64_t info = mine ? P.tmp[c][i] : 0;  // raw length 0 for rows that are not copied
        const uint64_t off = mine ? P.lens[(size_t)P.strk[c] * (P.nd + 1) + i] : 0;
        uint8_t *const base = P.bytes[c];
#pragma unroll 1
        for (uint32_t step = 0; step < 8; ++step) {
            const uint32_t src_lane = step * 4 + sub;
            const uint64_t ci = __shfl_sync(0xFFFFFFFFu, info, src_lane);
            const uint64_t co = __shfl_sync(0xFFFFFFFFu, off, src_lane);
            const uint32_t raw = (uint32_t)(ci >> 32) & 0x7FFFFFFFu;
            const uint8_t *src = P.buf + (uint32_t)ci;
            uint8_t *dst = base + co;
            if (!(ci >> 63)) {
                for (uint32_t k = k0; k < raw; k += 8) dst[k] = src[k];
            } else if (k0 == 0) {
                uint32_t o = 0;
                for (uint32_t k = 0; k < raw; ++k) {
                    if (src[k] == P.quote) {
                        ++k;
                        if (k >= raw) break;
                    }
                    dst[o++] = src[k];
                }
            }
        }
    }
}

// Validity words of the Option columns, in block (compacted) row order: one thread per block row reads its data row's null
// mask (csv_parse_one_row) and each warp ballots one word per column; bits past n_good are zero.
struct CsvValidParams {
    uint64_t n_good;
    uint32_t n_opt;
    const uint64_t *nullmask;  // [nd], per data row
    const uint32_t *rowmap;    // [n_good], block row -> data row
    uint8_t slot[TPLX_MAX_COLS];
    uint32_t *words[TPLX_MAX_COLS];
};
__global__ void __launch_bounds__(CSV_NT) csv_pack_valid(const CsvValidParams P) {
    const uint64_t pos = (uint64_t)blockIdx.x * CSV_NT + threadIdx.x;
    const uint64_t m = pos < P.n_good ? P.nullmask[P.rowmap[pos]] : ~0ull;
    const bool write = (threadIdx.x & 31) == 0 && (pos >> 5) < ((P.n_good + 31) >> 5);
    for (uint32_t k = 0; k < P.n_opt; ++k) {
        const uint32_t w = __ballot_sync(0xFFFFFFFFu, !((m >> P.slot[k]) & 1ull));
        if (write) P.words[k][pos >> 5] = w;
    }
}

// ---- K7: result columns -> CSV text (fast_csvwriter, PipelineBuilder.cc:1550-1722) ------------------------------
__global__ void __launch_bounds__(CSV_NT) csv_sink_sizes(const CsvSinkCols C, uint64_t n, uint64_t *__restrict__ sizes,
                                                         uint32_t *__restrict__ unsupported) {
    const uint64_t r = (uint64_t)blockIdx.x * CSV_NT + threadIdx.x;
    if (r >= n) return;
    const uint64_t l = csv_sink_row_len(C, r);
    if (!l) *unsupported = 1;  // an f64 cell beyond the exact-arithmetic range
    sizes[r] = l;
}
__global__ void __launch_bounds__(CSV_NT) csv_sink_write(const CsvSinkCols C, uint64_t n, const uint64_t *__restrict__ row_off,
                                                         uint8_t *__restrict__ out) {
    const uint64_t r = (uint64_t)blockIdx.x * CSV_NT + threadIdx.x;
    if (r < n) csv_sink_row_write(C, r, out + row_off[r]);
}

}  // namespace tplx
