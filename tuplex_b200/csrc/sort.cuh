// sort.cuh — K11, the device key sort (tplx_gpu_result_sort_by_keys): a stable order of row indices by a tuple of key columns, in
// the order the host path gives groups (dataset._key_order for columns of one type): None first, i64 signed, bool False first, str by
// bytes (a prefix first), the first key column most significant, equal keys in input order.
//
// Building block: a stable LSD radix pass over (u64 key, u32 row) pairs, one 8-bit digit per pass.
//   sort_keygen_kernel    key of every row of the current order, plus the AND and OR of all keys: a digit in which they agree is
//                         the same in every key, and its pass is skipped (small ranges cost few passes)
//   sort_count_kernel     per-tile digit counts, stored digit-major (counts[digit * n_tiles + tile])
//   device_scan           exclusive scan of the counts: where each (digit, tile) run starts
//   sort_scatter_kernel   tile-local stable ranks (warp __match_any_sync + per-warp digit counts), then the scatter
// Several key columns: the current order is sorted stably by each column, from the last key column to the first.
// Option columns: the values (None rows with a constant key), then one pass on the None flag puts None first.
// Strings: MSD refinement over 8-byte words (keyhash.cuh sort_str_word / sort_str_class). Round k sorts every row by
// (segment, word, class), where a segment holds rows still tied; rows with equal word and class 9 stay tied and go on to the next
// word. Before a round, a segment jumps ahead by the words all its members share with its first member (sort_lcp_kernel), so keys
// that share a long prefix take one round, not one per 8 bytes. Finished rows have a segment of their own and stay where they are.
#pragma once
#include <stdint.h>
#include "keyhash.cuh"

namespace tplx {

constexpr uint32_t SORT_NT = 256;
constexpr uint32_t SORT_IPT = 16;
constexpr uint32_t SORT_TILE = SORT_NT * SORT_IPT;

enum SortKeyKind : uint32_t { SK_I64 = 0, SK_BOOL = 1, SK_NONE = 2, SK_WORD = 3, SK_CLASS = 4, SK_SEG = 5 };

struct SortCol {
    const void *data;         // 8-byte values, or string bytes
    const uint32_t *offsets;  // strings: n + 1 offsets
    const uint32_t *valid;    // validity bitmap, or nullptr
};

// per-row state of the string refinement, indexed by row (seg_first and seg_skip by segment)
struct SortStr {
    uint32_t *depth;      // word the row compares next
    uint32_t *seg;        // segment of the row; segments are numbered in order
    uint32_t *seg_first;  // first row of every segment
    uint32_t *seg_skip;   // words every member of the segment shares with its first row
    uint8_t *active;      // the row is still tied with another
};

__device__ __forceinline__ bool sort_present(const uint32_t *valid, uint32_t r) {
    return !valid || ((__ldg(valid + (r >> 5)) >> (r & 31)) & 1u);
}

__device__ __forceinline__ void sort_str(const SortCol &c, uint32_t r, const uint8_t **p, uint32_t *len) {
    const uint32_t s0 = __ldg(c.offsets + r);
    *p = static_cast<const uint8_t *>(c.data) + s0;
    *len = sort_present(c.valid, r) ? __ldg(c.offsets + r + 1) - s0 : 0u;  // None sorts as the empty string, then the None pass
}

__device__ __forceinline__ uint64_t sort_key(uint32_t kind, const SortCol &c, const SortStr &S, uint32_t r) {
    switch (kind) {
        case SK_I64: return sort_present(c.valid, r) ? sort_key_i64((int64_t)__ldg(static_cast<const uint64_t *>(c.data) + r)) : 0;
        case SK_BOOL: return sort_present(c.valid, r) ? (__ldg(static_cast<const uint64_t *>(c.data) + r) != 0) : 0;
        case SK_NONE: return sort_present(c.valid, r) ? 1 : 0;
        case SK_SEG: return S.seg[r];
        default: {
            if (!S.active[r]) return 0;
            const uint8_t *p;
            uint32_t len;
            sort_str(c, r, &p, &len);
            return kind == SK_WORD ? sort_str_word(p, len, S.depth[r]) : sort_str_class(len, S.depth[r]);
        }
    }
}

__device__ __forceinline__ uint64_t warp_and64(uint64_t v) {
    for (int o = 16; o; o >>= 1) v &= __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}
__device__ __forceinline__ uint64_t warp_or64(uint64_t v) {
    for (int o = 16; o; o >>= 1) v |= __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

// keys[i] = key of row v[i]; andor[0] &= every key, andor[1] |= every key
__global__ void __launch_bounds__(SORT_NT) sort_keygen_kernel(uint32_t kind, SortCol c, SortStr S, const uint32_t *__restrict__ v, uint64_t n,
                                                               uint64_t *__restrict__ keys, unsigned long long *__restrict__ andor) {
    const uint64_t i = (uint64_t)blockIdx.x * SORT_NT + threadIdx.x;
    uint64_t a = ~0ull, o = 0;
    if (i < n) {
        const uint64_t k = sort_key(kind, c, S, v[i]);
        keys[i] = k;
        a = o = k;
    }
    a = warp_and64(a);
    o = warp_or64(o);
    if ((threadIdx.x & 31) == 0) {
        atomicAnd(andor, (unsigned long long)a);
        atomicOr(andor + 1, (unsigned long long)o);
    }
}

__global__ void __launch_bounds__(SORT_NT) sort_count_kernel(const uint64_t *__restrict__ keys, uint64_t n, uint32_t shift, uint32_t n_tiles,
                                                              uint64_t *__restrict__ counts) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t base = (uint64_t)blockIdx.x * SORT_TILE;
    for (uint32_t k = 0; k < SORT_IPT; ++k) {
        const uint64_t i = base + k * SORT_NT + threadIdx.x;
        if (i < n) atomicAdd(&h[(uint32_t)(keys[i] >> shift) & 255u], 1u);
    }
    __syncthreads();
    counts[(uint64_t)threadIdx.x * n_tiles + blockIdx.x] = h[threadIdx.x];
}

// Stable: the tile's items go in SORT_IPT rounds of SORT_NT consecutive items; an item's place is its digit's start for the tile,
// plus the items of that digit in earlier rounds, in earlier warps of this round, and in earlier lanes of its warp.
__global__ void __launch_bounds__(SORT_NT) sort_scatter_kernel(const uint64_t *__restrict__ kin, const uint32_t *__restrict__ vin, uint64_t n,
                                                                uint32_t shift, uint32_t n_tiles, const uint64_t *__restrict__ start,
                                                                uint64_t *__restrict__ kout, uint32_t *__restrict__ vout) {
    constexpr uint32_t NW = SORT_NT / 32;
    __shared__ uint64_t base[256];
    __shared__ uint32_t wcnt[NW][256];
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    base[t] = start[(uint64_t)t * n_tiles + blockIdx.x];
    for (uint32_t w = 0; w < NW; ++w) wcnt[w][t] = 0;
    __syncthreads();
    const uint64_t tile0 = (uint64_t)blockIdx.x * SORT_TILE;
    for (uint32_t k = 0; k < SORT_IPT; ++k) {
        const uint64_t i = tile0 + k * SORT_NT + t;
        const bool ok = i < n;
        const uint64_t key = ok ? kin[i] : 0;
        const uint32_t d = ok ? ((uint32_t)(key >> shift) & 255u) : 256u;
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
        const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
        if (ok && rank == 0) wcnt[warp][d] = __popc(peers);
        __syncthreads();
        if (ok) {
            uint64_t pos = base[d] + rank;
            for (uint32_t w = 0; w < warp; ++w) pos += wcnt[w][d];
            kout[pos] = key;
            vout[pos] = vin[i];
        }
        __syncthreads();
        uint32_t tot = 0;
        for (uint32_t w = 0; w < NW; ++w) {
            tot += wcnt[w][t];
            wcnt[w][t] = 0;
        }
        base[t] += tot;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(SORT_NT) sort_iota_kernel(uint32_t *__restrict__ v, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * SORT_NT + threadIdx.x;
    if (i < n) v[i] = (uint32_t)i;
}

// Words an active row shares with its segment's first row from its depth on, both with class 9; the segment skips the least of them.
__global__ void __launch_bounds__(SORT_NT) sort_lcp_kernel(SortCol c, SortStr S, uint64_t n) {
    const uint64_t r = (uint64_t)blockIdx.x * SORT_NT + threadIdx.x;
    if (r >= n || !S.active[r]) return;
    const uint32_t s = S.seg[r], f = S.seg_first[s], k = S.depth[r];
    const uint8_t *pr, *pf;
    uint32_t lr, lf;
    sort_str(c, (uint32_t)r, &pr, &lr);
    sort_str(c, f, &pf, &lf);
    uint32_t w = 0;
    while (sort_str_class(lr, k + w) == 9 && sort_str_class(lf, k + w) == 9 && sort_str_word(pr, lr, k + w) == sort_str_word(pf, lf, k + w)) ++w;
    atomicMin(S.seg_skip + s, w);
}

__global__ void __launch_bounds__(SORT_NT) sort_skip_kernel(SortStr S, uint64_t n) {
    const uint64_t r = (uint64_t)blockIdx.x * SORT_NT + threadIdx.x;
    if (r < n && S.active[r]) S.depth[r] += S.seg_skip[S.seg[r]];
}

// after a round's sort: tied[j] = the row at position j stays tied with the one before it (same segment, word and class, class 9);
// flags[j] = a segment starts at j
__global__ void __launch_bounds__(SORT_NT) sort_tie_kernel(SortCol c, SortStr S, const uint32_t *__restrict__ v, uint64_t n,
                                                            uint8_t *__restrict__ tied, uint64_t *__restrict__ flags) {
    const uint64_t j = (uint64_t)blockIdx.x * SORT_NT + threadIdx.x;
    if (j >= n) return;
    bool t = false;
    if (j > 0) {
        const uint32_t r = v[j], p = v[j - 1];
        if (S.active[r] && S.active[p] && S.seg[r] == S.seg[p]) {
            const uint8_t *pr, *pp;
            uint32_t lr, lp;
            sort_str(c, r, &pr, &lr);
            sort_str(c, p, &pp, &lp);
            const uint32_t k = S.depth[r];
            t = sort_str_class(lr, k) == 9 && sort_str_class(lp, k) == 9 && sort_str_word(pr, lr, k) == sort_str_word(pp, lp, k);
        }
    }
    tied[j] = t;
    flags[j] = t ? 0 : 1;
}

// segments of the next round from the scanned flags; a row stays active when it is tied with a neighbour, and moves to its next word
__global__ void __launch_bounds__(SORT_NT) sort_assign_kernel(SortStr S, const uint32_t *__restrict__ v, uint64_t n, const uint8_t *__restrict__ tied,
                                                               const uint64_t *__restrict__ ex, unsigned long long *__restrict__ n_active) {
    const uint64_t j = (uint64_t)blockIdx.x * SORT_NT + threadIdx.x;
    bool act = false;
    if (j < n) {
        const uint32_t r = v[j];
        const uint32_t s = (uint32_t)(tied[j] ? ex[j] - 1 : ex[j]);
        S.seg[r] = s;
        if (!tied[j]) S.seg_first[s] = r;
        act = tied[j] || (j + 1 < n && tied[j + 1]);
        S.active[r] = act;
        if (act) S.depth[r] += 1;
    }
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, act);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_active, (unsigned long long)__popc(b));
}

}  // namespace tplx
