// text.cuh — K10: text file bytes -> one string column (a line per row), on the device.
//
// Replaces the host reader of Context.text (and the reference's TextReader, core/src/physical/TextReader.cc:60-140, in front
// of a TransformStage). Semantics live in textops.cuh. The input is a CSV upload buffer (tplx_gpu_csv_upload): n data bytes,
// '\n' at [n], zero padding to a 16 KB tile.
//   1. text_tile_counts   per 16 KB tile: line ends (popcount of the '\n' lanes of each word) and whether it holds a byte
//                         >= 0x80
//   2. device_scan        exclusive scan of the tile counts: lines before each tile
//   3. text_line_ends     the same walk with a block scan of the thread counts: the position of every line end
//   4. text_line_info     one thread per line: '\r' trim, length after the UTF-8 replacement (a line whose tiles are all
//                         ASCII skips validation), null flag, good flag
//   5. device_scan_batched   output offsets and block positions of the lines, one batched scan
//   6. text_copy_lines    one warp per 32 lines: offsets, rowmap and bad rows from lane i, then every line's bytes copied by
//                         the whole warp (consecutive lanes on consecutive bytes); a line with invalid UTF-8 is written
//                         replaced by its first lane
//   7. text_pack_valid    Option[str] only: validity words by ballot, in block row order
// HBM-bound byte work. Algorithmic traffic per input byte: read 3x (steps 1, 3, 6; step 4 touches the bytes of non-ASCII and
// short null candidate lines only) + written once, plus 4 B of line end, 17 B of per-line scratch and 8 B of offsets + rowmap
// per line.
#pragma once
#include <stdint.h>
#include "textops.cuh"
#include "../../include/tplx_gpu.h"

namespace tplx {

constexpr int TEXT_NT = 256;
constexpr uint32_t TEXT_TILE = TEXT_NT * TEXT_SPAN;  // 16 KB per CTA, the CSV upload buffer's padding unit

// exclusive block scan (TEXT_NT threads) of one count per thread; *total = the block's sum
__device__ __forceinline__ uint32_t text_block_scan(uint32_t v, uint32_t *total) {
    __shared__ uint32_t warp_tot[TEXT_NT / 32];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t a = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (lane >= (uint32_t)o) inc += a;
    }
    if (lane == 31) warp_tot[wid] = inc;
    __syncthreads();
    uint32_t pre = 0, tot = 0;
    for (uint32_t w = 0; w < TEXT_NT / 32; ++w) {
        if (w < wid) pre += warp_tot[w];
        tot += warp_tot[w];
    }
    __syncthreads();
    *total = tot;
    return pre + inc - v;
}

__global__ void __launch_bounds__(TEXT_NT) text_tile_counts(const uint8_t *__restrict__ buf, uint64_t n, uint64_t *__restrict__ counts,
                                                            uint8_t *__restrict__ tile_ascii) {
    const uint64_t start = (uint64_t)blockIdx.x * TEXT_TILE + (uint64_t)threadIdx.x * TEXT_SPAN;
    bool ascii = true;
    const uint32_t c = text_walk_span(buf, start, n, &ascii, [](uint64_t) {});
    uint32_t tot;
    text_block_scan(c, &tot);
    const int all_ascii = __syncthreads_and(ascii ? 1 : 0);
    if (threadIdx.x == 0) {
        counts[blockIdx.x] = tot;
        tile_ascii[blockIdx.x] = all_ascii ? 1 : 0;
    }
}

__global__ void __launch_bounds__(TEXT_NT) text_line_ends(const uint8_t *__restrict__ buf, uint64_t n, const uint64_t *__restrict__ tile_start,
                                                          uint32_t *__restrict__ ends) {
    const uint64_t start = (uint64_t)blockIdx.x * TEXT_TILE + (uint64_t)threadIdx.x * TEXT_SPAN;
    bool ascii = true;
    const uint32_t c = text_walk_span(buf, start, n, &ascii, [](uint64_t) {});
    uint32_t tot;
    uint64_t line = tile_start[blockIdx.x] + text_block_scan(c, &tot);
    if (!c) return;
    text_walk_span(buf, start, n, &ascii, [&](uint64_t pos) { ends[line++] = (uint32_t)pos; });
}

struct TextParams {
    const uint8_t *buf;
    const uint32_t *ends;       // [nl]
    const uint8_t *tile_ascii;  // [tiles]
    uint32_t nl;
    uint8_t option;             // 1: a null line is None (good, empty, null flag); 0: it is a bad row (NULLERROR)
    CsvNulls nulls;
    uint64_t *lens;             // [2][nl + 1]: output bytes, then good flags; scanned in place by step 5
    uint8_t *flags;             // [nl]: TEXT_F_* bits
};
constexpr uint8_t TEXT_F_VERBATIM = 1, TEXT_F_NULL = 2;

__global__ void __launch_bounds__(TEXT_NT) text_line_info(const TextParams P) {
    const uint32_t i = blockIdx.x * TEXT_NT + threadIdx.x;
    if (i >= P.nl) return;
    uint32_t s, e;
    text_line_range(P.buf, P.ends, i, &s, &e);
    bool ascii = true;
    if (e > s)
        for (uint32_t t = s / TEXT_TILE; t <= (e - 1) / TEXT_TILE && ascii; ++t) ascii = P.tile_ascii[t] != 0;
    bool replaced = false;
    const uint64_t out = ascii ? (uint64_t)(e - s) : text_replaced_len(P.buf + s, e - s, &replaced);
    const bool null = P.nulls.n && out <= 64 && text_is_null(P.buf + s, e - s, !replaced, out, P.nulls);
    const bool good = P.option || !null;
    P.lens[i] = (good && !null) ? out : 0;
    P.lens[(size_t)P.nl + 1 + i] = good ? 1 : 0;
    P.flags[i] = (replaced ? 0 : TEXT_F_VERBATIM) | (null ? TEXT_F_NULL : 0);
}

struct TextCopyParams {
    const uint8_t *buf;
    const uint32_t *ends;
    const uint8_t *flags;
    const uint64_t *off;   // scanned output bytes, [nl] = total
    const uint64_t *pos;   // scanned good flags, [nl] = n_good
    uint32_t nl;
    uint8_t *bytes;
    uint32_t *offsets;     // [n_good + 1]
    uint32_t *rowmap;      // [n_good]: block row -> line
    tplx_csv_bad_row *bad; // [nl - n_good]
};

__global__ void __launch_bounds__(TEXT_NT) text_copy_lines(const TextCopyParams P) {
    const uint32_t g = (blockIdx.x * TEXT_NT + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t first = g * 32;
    if (first >= P.nl) return;
    const uint32_t i = first + lane;
    uint32_t s = 0, e = 0, copy = 0;
    uint64_t o = 0;
    uint8_t f = 0;
    if (i < P.nl) {
        text_line_range(P.buf, P.ends, i, &s, &e);
        const uint64_t pos = P.pos[i];
        f = P.flags[i];
        o = P.off[i];
        if (P.pos[i + 1] != pos) {  // good line: block row pos
            P.offsets[pos] = (uint32_t)o;
            P.rowmap[pos] = i;
            if (pos + 1 == P.pos[P.nl]) P.offsets[pos + 1] = (uint32_t)P.off[P.nl];
            copy = (f & TEXT_F_NULL) ? 0u : 1u;
        } else {
            tplx_csv_bad_row b;
            b.row = i;
            b.code = TPLX_EC_NULLERROR;
            b.line_start = i == 0 ? 0u : P.ends[i - 1] + 1;
            b.line_end = P.ends[i];
            P.bad[i - pos] = b;
        }
    }
#pragma unroll 1
    for (uint32_t j = 0; j < 32; ++j) {
        const uint32_t cj = __shfl_sync(0xFFFFFFFFu, copy, j);
        if (!cj) continue;
        const uint32_t sj = __shfl_sync(0xFFFFFFFFu, s, j), ej = __shfl_sync(0xFFFFFFFFu, e, j);
        const uint64_t oj = __shfl_sync(0xFFFFFFFFu, o, j);
        const uint32_t fj = __shfl_sync(0xFFFFFFFFu, (uint32_t)f, j);
        const uint8_t *src = P.buf + sj;
        uint8_t *dst = P.bytes + oj;
        if (fj & TEXT_F_VERBATIM) {
            for (uint32_t k = lane; k < ej - sj; k += 32) dst[k] = src[k];
        } else if (lane == 0) {
            uint64_t w = 0;
            text_replaced_emit(src, ej - sj, [&](uint8_t b) { dst[w++] = b; });
        }
    }
}

// validity words of the Option[str] column: every line is a block row (nothing is bad in that mode), bit clear = None
__global__ void __launch_bounds__(TEXT_NT) text_pack_valid(const uint8_t *__restrict__ flags, uint64_t n, uint32_t *__restrict__ words) {
    const uint64_t r = (uint64_t)blockIdx.x * TEXT_NT + threadIdx.x;
    const bool present = r < n && !(flags[r] & TEXT_F_NULL);
    const uint32_t w = __ballot_sync(0xFFFFFFFFu, present);
    if ((threadIdx.x & 31) == 0 && (r >> 5) < ((n + 31) >> 5)) words[r >> 5] = w;
}

}  // namespace tplx
