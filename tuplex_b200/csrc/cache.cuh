// cache.cuh — what DataSet.cache() does to the rows it keeps on the device: column statistics of a block, and the UTF-8 rewrite of
// the ranged, typed concatenation (concat.cuh, tplx_gpu_block_concat_pieces).
//
// A cached dataset must be the dataset the host would build from the same rows (Context._source_from_rows over the Python values
// of the rows): a column without None in any row is plain T, one that is None in every row is an i64 placeholder column, and a
// string that is not valid UTF-8 is stored as bytes.decode("utf-8", "replace").encode(). The statistics decide this per column:
//   cache_stats_kernel   one CTA per (CACHE_TILE_ROWS rows, column): None rows = cleared validity bits within [0, n_rows) (tail
//                        bits of result blocks may be garbage and are masked); strings that change under the replacement, validated
//                        only in tiles whose bytes hold a byte >= 0x80 (the tile's bytes are read once, word by word, like
//                        K10's text_tile_counts)
// The rewrite of a string column over the pieces of a concatenation:
//   cache_utf8_len_kernel   one thread per output row: its length after the replacement
//   device_scan             exclusive scan: output offsets, total at [n]
//   cache_utf8_copy_kernel  one thread per output row: its bytes after the replacement (valid characters are copied as they are)
// The per-row functions are host-compilable: tests/cache_host.cpp runs the same three steps on the CPU.
#pragma once
#include <stdint.h>
#include "textops.cuh"

namespace tplx {

// bytes of string s of a column (bytes, offsets) after the replacement
TPLX_HD uint64_t cache_utf8_len(const uint8_t *bytes, const uint32_t *offsets, uint64_t s) {
    bool replaced;
    return text_replaced_len(bytes + offsets[s], offsets[s + 1] - offsets[s], &replaced);
}

// string s of a column written at out after the replacement
TPLX_HD void cache_utf8_write(const uint8_t *bytes, const uint32_t *offsets, uint64_t s, uint8_t *out) {
    uint64_t w = 0;
    text_replaced_emit(bytes + offsets[s], offsets[s + 1] - offsets[s], [&](uint8_t b) { out[w++] = b; });
}

// does string s change under the replacement?
TPLX_HD bool cache_utf8_invalid(const uint8_t *bytes, const uint32_t *offsets, uint64_t s) {
    bool replaced;
    text_replaced_len(bytes + offsets[s], offsets[s + 1] - offsets[s], &replaced);
    return replaced;
}

#ifdef __CUDACC__
}  // namespace tplx
#include "concat.cuh"
#include "../../include/tplx_gpu.h"
namespace tplx {

constexpr uint32_t CACHE_NT = 256;
constexpr uint32_t CACHE_TILE_ROWS = 4 * CACHE_NT;  // rows per CTA of the statistics

struct StatsCol {
    uint8_t type;
    const uint8_t *bytes;     // string column: bytes and n_rows + 1 offsets
    const uint32_t *offsets;
    const uint32_t *valid;    // validity words, or nullptr
};

// counts[2c] += None rows, counts[2c + 1] += strings changed by the replacement, over the rows of tile blockIdx.x of column
// blockIdx.y
__global__ void __launch_bounds__(CACHE_NT) cache_stats_kernel(const StatsCol *__restrict__ cols, uint64_t n,
                                                               unsigned long long *__restrict__ counts) {
    const StatsCol c = cols[blockIdx.y];
    const uint64_t r0 = (uint64_t)blockIdx.x * CACHE_TILE_ROWS;
    const uint64_t r1 = r0 + CACHE_TILE_ROWS < n ? r0 + CACHE_TILE_ROWS : n;
    if (c.valid && threadIdx.x < CACHE_TILE_ROWS / 32) {
        const uint64_t w = (r0 >> 5) + threadIdx.x;
        uint32_t none = 0;
        if (w * 32 < r1) {
            const uint64_t rows = r1 - w * 32 < 32 ? r1 - w * 32 : 32;
            const uint32_t mask = rows == 32 ? 0xFFFFFFFFu : ((1u << rows) - 1u);
            none = (uint32_t)__popc(~c.valid[w] & mask);
        }
        for (int o = 16; o; o >>= 1) none += __shfl_xor_sync(0xFFFFFFFFu, none, o);
        if (threadIdx.x == 0 && none) atomicAdd(&counts[2 * blockIdx.y], (unsigned long long)none);
    }
    if (c.type != TPLX_T_STR) return;
    // ASCII test of the tile's bytes [offsets[r0], offsets[r1]), by aligned 8-byte words (the words may take in bytes of the
    // neighbouring rows: a false "not ASCII" only costs the validation below)
    const uint64_t b0 = c.offsets[r0], b1 = c.offsets[r1];
    const uintptr_t a0 = ((uintptr_t)(c.bytes + b0)) & ~(uintptr_t)7, a1 = (uintptr_t)(c.bytes + b1);
    bool high = false;
    for (uintptr_t a = a0 + 8 * threadIdx.x; a < a1; a += 8 * CACHE_NT)
        high = high || (*reinterpret_cast<const uint64_t *>(a) & 0x8080808080808080ull) != 0;
    if (!__syncthreads_or(high ? 1 : 0)) return;
    uint32_t bad = 0;
    for (uint64_t r = r0 + threadIdx.x; r < r1; r += CACHE_NT) bad += cache_utf8_invalid(c.bytes, c.offsets, r) ? 1u : 0u;
    if (bad) atomicAdd(&counts[2 * blockIdx.y + 1], (unsigned long long)bad);
}

// lens[i] = bytes of output row i after the replacement (i < n)
__global__ void __launch_bounds__(CACHE_NT) cache_utf8_len_kernel(const ConcatPart *__restrict__ parts, const uint64_t *__restrict__ row_base,
                                                                  uint32_t n_parts, uint64_t n, uint64_t *__restrict__ lens) {
    const uint64_t i = (uint64_t)blockIdx.x * CACHE_NT + threadIdx.x;
    if (i >= n) return;
    const uint32_t p = concat_part_of(row_base, n_parts, i);
    lens[i] = cache_utf8_len(parts[p].bytes, parts[p].offsets, parts[p].row0 + i - row_base[p]);
}

// output offsets (from the scanned lengths, total at pos[n]) and bytes of every output row
__global__ void __launch_bounds__(CACHE_NT) cache_utf8_copy_kernel(const ConcatPart *__restrict__ parts, const uint64_t *__restrict__ row_base,
                                                                   uint32_t n_parts, uint64_t n, const uint64_t *__restrict__ pos,
                                                                   uint32_t *__restrict__ offsets, uint8_t *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * CACHE_NT + threadIdx.x;
    if (i > n) return;
    offsets[i] = (uint32_t)pos[i];
    if (i == n) return;
    const uint32_t p = concat_part_of(row_base, n_parts, i);
    cache_utf8_write(parts[p].bytes, parts[p].offsets, parts[p].row0 + i - row_base[p], out + pos[i]);
}
#endif

}  // namespace tplx
