// concat.cuh — block concatenation: row ranges of several device blocks, in order, as one block (tplx_gpu_block_concat_pieces;
// tplx_gpu_block_concat takes whole blocks).
//
// Used where one operator needs a single block of rows that an upstream stage produced as several block results (the build side
// of a hash join, K8, takes exactly one block). Fixed-width columns and string bytes move with device-to-device copies; what
// has to be rewritten per row runs as one batched launch per column over all parts:
//   - string offsets: row i of part p gets its offset less the part's first offset plus the bytes of the parts in front of p;
//   - validity words: every output word is assembled from the (at most a few) parts whose rows it covers, each part's words
//     realigned from the part's first row to its first output row with a funnel shift. Bits past a part's row count are never read into the
//     output (results may carry garbage there); a part without a bitmap contributes set bits; the output's tail bits are zero.
#pragma once
#include <stdint.h>

namespace tplx {

// per (column, part) of a concat; a part is rows [row0, row0 + its row count) of a block
struct ConcatPart {
    const uint8_t *bytes;     // string column: the block's bytes
    const uint32_t *offsets;  // string column: the block's offsets
    const uint32_t *valid;    // validity words of the block, or nullptr (every row holds a value)
    uint64_t row0;            // the part's first row in the block
    uint64_t byte_base;       // string column: output position of the part's first byte
    uint64_t shift;           // string column: byte_base - offsets[row0], modulo 2^64
};

constexpr uint32_t CONCAT_NT = 256;

// last part p with row_base[p] <= r (row_base[0] = 0, ascending, n_parts + 1 entries): the part that holds output row r when
// r < row_base[n_parts]; empty parts are skipped because row_base[p + 1] > r for the part returned
__device__ __forceinline__ uint32_t concat_part_of(const uint64_t *__restrict__ row_base, uint32_t n_parts, uint64_t r) {
    uint32_t lo = 0, hi = n_parts;  // answer in [0, n_parts)
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (row_base[mid] <= r) lo = mid;
        else hi = mid;
    }
    return lo;
}

// out[0 .. n]: row offsets of the concatenated string column; out[n] = total bytes
__global__ void __launch_bounds__(CONCAT_NT) concat_offsets_kernel(const ConcatPart *__restrict__ parts, const uint64_t *__restrict__ row_base,
                                                                  uint32_t n_parts, uint64_t n, uint64_t total, uint32_t *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * CONCAT_NT + threadIdx.x;
    if (i > n) return;
    if (i == n) {
        out[n] = (uint32_t)total;
        return;
    }
    const uint32_t p = concat_part_of(row_base, n_parts, i);
    const ConcatPart cp = parts[p];
    out[i] = (uint32_t)(cp.offsets[cp.row0 + i - row_base[p]] + cp.shift);
}

// out[w] for w < (n + 31) / 32: bits 32w .. 32w + 31 of the concatenated column's validity
__global__ void __launch_bounds__(CONCAT_NT) concat_valid_kernel(const ConcatPart *__restrict__ parts, const uint64_t *__restrict__ row_base,
                                                                uint32_t n_parts, uint64_t n, uint32_t *__restrict__ out) {
    const uint64_t w = (uint64_t)blockIdx.x * CONCAT_NT + threadIdx.x;
    const uint64_t r0 = w * 32;
    if (r0 >= n) return;
    const uint64_t r1 = r0 + 32 < n ? r0 + 32 : n;  // output rows [r0, r1) of this word
    uint32_t word = 0;
    for (uint32_t p = concat_part_of(row_base, n_parts, r0); p < n_parts && row_base[p] < r1; ++p) {
        const uint64_t b = row_base[p], e = row_base[p + 1];
        if (e <= r0 || e == b) continue;  // a part in front of the word, or an empty part inside it (no rows, no words to read)
        const uint64_t lo = (r0 > b ? r0 : b) - b, hi = (r1 < e ? r1 : e) - b;  // part rows [lo, hi), 1..32 of them
        const uint32_t cnt = (uint32_t)(hi - lo);
        const uint32_t mask = cnt == 32 ? 0xFFFFFFFFu : ((1u << cnt) - 1u);
        const uint32_t *v = parts[p].valid;
        uint32_t bits = mask;
        if (v) {
            const uint64_t sl = parts[p].row0 + lo, sh = parts[p].row0 + hi - 1;  // the block's rows
            const uint64_t wl = sl >> 5, wh = sh >> 5;  // the block's words that hold them (one or two)
            const uint32_t a = v[wl], c = wh != wl ? v[wh] : 0u;
            bits = __funnelshift_r(a, c, (uint32_t)(sl & 31)) & mask;
        }
        word |= bits << (uint32_t)(b + lo - r0);
    }
    out[w] = word;
}

}  // namespace tplx
