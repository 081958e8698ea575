// join.cuh — K8: hash-join build + probe between two column blocks (SURVEY §8f rank 3).
//
// Replaces, for the normal case, the reference's hash-join pair of stages:
//   build side  — a TransformStage with a hash-table endpoint: every row is appended to the bucket of its key
//                 (writeRowToHashTable, tuplex/core/src/physical/TransformTask.cc:769-842; buckets keep rows in
//                 insertion order = input order; rows with a NULL key go to the null bucket, :776-789);
//   probe side  — addHashJoinProbe in the row pipeline (tuplex/core/src/physical/PipelineBuilder.cc:2330-2523): look the
//                 key up, then loop over the bucket (createInnerJoinBucketLoop :2110-2212 / createLeftJoinBucketLoop
//                 :2214-2328) and emit one combined row per bucket row, in bucket order; a left join emits the probe row
//                 once with NULL build columns when nothing matches.
// Output row order is therefore: probe rows in input order, matches of one probe row in build-row order. It is part of
// the contract (tuplex/test/core/JoinTest.cc:135-170) and is what the kernels below produce, deterministically.
//
// Device design. The reference serialises each build row into a malloc'd, realloc-grown bucket; here the build side stays
// columnar and the table holds only row numbers:
//   slots[cap]      open addressing, value = representative build row + 1 of the key that owns the slot (0 = empty). Keys are
//                   compared against the immutable build key column, so claiming a slot is ONE atomicCAS and needs no
//                   "busy" state;
//   start[cap + 2]  CSR offsets of the groups (group id = slot index; group `cap` is the null bucket);
//   rows[n_build]   build rows grouped by key, ascending inside a group (filled with atomics, then every group with more
//                   than one row is put in order: thread-per-group insertion sort, CTA-per-group counting rank for
//                   groups above 32 rows).
// Probe = two passes over the probe block (count, exclusive scan, emit) giving (probe row, build row) index pairs in the
// output order above, then a columnar gather of every output column (gather.cuh) with validity bitmaps where a column is nullable.
// The probe is HBM-latency work (one random slot + one random key read per probe row): 256-thread CTAs, grid sized to the
// block, every lane independent; bucket loops of 32+ rows are taken by the whole warp.
#pragma once
#include <stdint.h>
#include "kernels.cuh"
#include "keyhash.cuh"

namespace tplx {

constexpr uint32_t JOIN_NONE = 0xFFFFFFFFu;
constexpr uint32_t JOIN_NT = 256;
constexpr uint32_t JOIN_SMALL = 32;  // groups up to this size are ordered by one thread

struct JoinKey {            // a key column (build or probe side)
    const void *data;       // 8-byte values, or string bytes
    const uint32_t *offsets;
    const uint32_t *valid;  // optional bitmap: bit (r & 31) of word r >> 5 set = value present
    uint32_t type;          // tplx_type
    uint32_t pad;
};

struct JoinTableDev {
    uint32_t *slots;   // cap
    uint64_t *start;   // cap + 2: exclusive scan of the group sizes (entry cap + 1 = n_build)
    uint32_t *rows;    // n_build
    uint64_t cap, mask;
    JoinKey key;       // the build side's key column (borrowed: the build block outlives the table)
};

__device__ __forceinline__ bool join_is_null(const JoinKey &k, uint64_t r) {
    return k.valid && !((k.valid[r >> 5] >> (r & 31)) & 1u);
}

__device__ __forceinline__ uint64_t join_hash(const JoinKey &k, uint64_t r) {
    if (k.type == TPLX_T_STR) {
        const uint32_t o0 = k.offsets[r], o1 = k.offsets[r + 1];
        return key_hash_bytes(reinterpret_cast<const uint8_t *>(k.data) + o0, o1 - o0);
    }
    return key_hash_i64(reinterpret_cast<const uint64_t *>(k.data)[r]);
}

__device__ __forceinline__ bool join_key_equal(const JoinKey &a, uint64_t ra, const JoinKey &b, uint64_t rb) {
    if (a.type == TPLX_T_STR) {
        const uint32_t a0 = a.offsets[ra], a1 = a.offsets[ra + 1], b0 = b.offsets[rb], b1 = b.offsets[rb + 1];
        if (a1 - a0 != b1 - b0) return false;
        const uint8_t *pa = reinterpret_cast<const uint8_t *>(a.data) + a0, *pb = reinterpret_cast<const uint8_t *>(b.data) + b0;
        for (uint32_t i = 0; i < a1 - a0; ++i)
            if (pa[i] != pb[i]) return false;
        return true;
    }
    return reinterpret_cast<const uint64_t *>(a.data)[ra] == reinterpret_cast<const uint64_t *>(b.data)[rb];
}

// ---- build -----------------------------------------------------------------------------------------------------------------
// one thread per build row: find or claim the slot of its key, count the row in its group
__global__ void __launch_bounds__(JOIN_NT) join_insert_kernel(JoinTableDev T, uint64_t n, uint32_t *__restrict__ row_group, uint64_t *__restrict__ cnt) {
    const uint64_t r = (uint64_t)blockIdx.x * JOIN_NT + threadIdx.x;
    if (r >= n) return;
    uint64_t g;
    if (join_is_null(T.key, r)) {
        g = T.cap;  // null bucket (TransformTask.cc:776-789)
    } else {
        uint64_t idx = (join_hash(T.key, r) >> 17) & T.mask;
        while (true) {
            uint32_t v = T.slots[idx];
            if (v == 0) {
                v = atomicCAS(&T.slots[idx], 0u, (uint32_t)r + 1u);
                if (v == 0) break;  // claimed: this row represents the key
            }
            if (join_key_equal(T.key, v - 1, T.key, r)) break;
            idx = (idx + 1) & T.mask;  // load <= 0.5: an empty slot always exists
        }
        g = idx;
    }
    row_group[r] = (uint32_t)g;
    atomicAdd((unsigned long long *)&cnt[g], 1ull);
}

// one thread per build row: place the row in its group's range (any order; join_order_* sort the ranges afterwards)
__global__ void __launch_bounds__(JOIN_NT) join_fill_kernel(JoinTableDev T, uint64_t n, const uint32_t *__restrict__ row_group, uint32_t *__restrict__ cursor) {
    const uint64_t r = (uint64_t)blockIdx.x * JOIN_NT + threadIdx.x;
    if (r >= n) return;
    const uint32_t g = row_group[r];
    const uint32_t k = atomicAdd(&cursor[g], 1u);
    T.rows[T.start[g] + k] = (uint32_t)r;
}

// one thread per group: ascending build-row order inside the bucket; groups above JOIN_SMALL rows are queued for a CTA
__global__ void __launch_bounds__(JOIN_NT) join_order_small_kernel(JoinTableDev T, uint32_t *__restrict__ big_list, uint32_t *__restrict__ n_big) {
    const uint64_t g = (uint64_t)blockIdx.x * JOIN_NT + threadIdx.x;
    if (g > T.cap) return;
    const uint64_t s = T.start[g], k = T.start[g + 1] - s;
    if (k < 2) return;
    if (k > JOIN_SMALL) {
        big_list[atomicAdd(n_big, 1u)] = (uint32_t)g;
        return;
    }
    uint32_t *a = T.rows + s;
    for (uint32_t i = 1; i < (uint32_t)k; ++i) {  // insertion sort, k <= 32
        const uint32_t v = a[i];
        uint32_t j = i;
        while (j > 0 && a[j - 1] > v) {
            a[j] = a[j - 1];
            --j;
        }
        a[j] = v;
    }
}

// one CTA per large group: rank of a row = number of rows of the group below it (rows are distinct), tiles through shared memory
__global__ void __launch_bounds__(JOIN_NT) join_order_big_kernel(JoinTableDev T, const uint32_t *__restrict__ big_list, uint32_t *__restrict__ tmp) {
    __shared__ uint32_t tile[2048];
    const uint32_t g = big_list[blockIdx.x];
    const uint64_t s = T.start[g], k = T.start[g + 1] - s;
    const uint32_t *a = T.rows + s;
    uint32_t *out = tmp + s;
    for (uint64_t i0 = 0; i0 < k; i0 += JOIN_NT) {
        const uint64_t i = i0 + threadIdx.x;
        const uint32_t v = i < k ? a[i] : 0u;
        uint64_t rank = 0;
        for (uint64_t j0 = 0; j0 < k; j0 += 2048) {
            __syncthreads();
            for (uint32_t t = threadIdx.x; t < 2048; t += JOIN_NT) tile[t] = j0 + t < k ? a[j0 + t] : 0xFFFFFFFFu;
            __syncthreads();
            for (uint32_t t = 0; t < 2048; ++t) rank += tile[t] < v;
        }
        if (i < k) out[rank] = v;
    }
}
__global__ void __launch_bounds__(JOIN_NT) join_copy_big_kernel(JoinTableDev T, const uint32_t *__restrict__ big_list, const uint32_t *__restrict__ tmp) {
    const uint32_t g = big_list[blockIdx.x];
    const uint64_t s = T.start[g], k = T.start[g + 1] - s;
    for (uint64_t i = threadIdx.x; i < k; i += JOIN_NT) T.rows[s + i] = tmp[s + i];
}

// ---- probe -----------------------------------------------------------------------------------------------------------------
// pass 1, one thread per probe row: group of its key (or none) and how many output rows it produces
__global__ void __launch_bounds__(JOIN_NT) join_probe_count_kernel(JoinTableDev T, JoinKey pk, uint64_t n, uint32_t left_outer,
                                                                   uint32_t *__restrict__ grp, uint64_t *__restrict__ cnt) {
    const uint64_t r = (uint64_t)blockIdx.x * JOIN_NT + threadIdx.x;
    if (r >= n) return;
    uint64_t g = JOIN_NONE;
    if (join_is_null(pk, r)) {
        g = T.cap;  // NULL matches NULL: the null bucket (JoinTest.cc:21-76)
    } else {
        uint64_t idx = (join_hash(pk, r) >> 17) & T.mask;
        while (true) {
            const uint32_t v = T.slots[idx];
            if (v == 0) break;
            if (join_key_equal(T.key, v - 1, pk, r)) {
                g = idx;
                break;
            }
            idx = (idx + 1) & T.mask;
        }
    }
    uint64_t k = 0;
    if (g != JOIN_NONE) k = T.start[g + 1] - T.start[g];
    if (k == 0) g = JOIN_NONE;
    grp[r] = (uint32_t)g;
    cnt[r] = k ? k : (left_outer ? 1 : 0);
}

// pass 2: write the (probe row, build row) pairs of every probe row at its scanned position; buckets of 32+ rows are
// written by the whole warp (coalesced), shorter ones by the row's own lane
__global__ void __launch_bounds__(JOIN_NT) join_probe_emit_kernel(JoinTableDev T, uint64_t n, const uint32_t *__restrict__ grp,
                                                                  const uint64_t *__restrict__ out_start, uint32_t *__restrict__ out_probe,
                                                                  uint32_t *__restrict__ out_build) {
    const uint64_t r = (uint64_t)blockIdx.x * JOIN_NT + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    uint32_t g = JOIN_NONE;
    uint64_t base = 0, k = 0, s = 0;
    if (r < n) {
        g = grp[r];
        base = out_start[r];
        k = out_start[r + 1] - base;
        if (g != JOIN_NONE) s = T.start[g];
    }
    const bool wide = g != JOIN_NONE && k >= 32;
    if (!wide) {
        if (g == JOIN_NONE) {
            if (k) {  // left join without a match: one row, build side NULL
                out_probe[base] = (uint32_t)r;
                out_build[base] = JOIN_NONE;
            }
        } else {
            for (uint64_t j = 0; j < k; ++j) {
                out_probe[base + j] = (uint32_t)r;
                out_build[base + j] = T.rows[s + j];
            }
        }
    }
    uint32_t m = __ballot_sync(0xFFFFFFFFu, wide);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const uint64_t rb = __shfl_sync(0xFFFFFFFFu, base, src), rk = __shfl_sync(0xFFFFFFFFu, k, src), rs = __shfl_sync(0xFFFFFFFFu, s, src);
        const uint32_t rr = (uint32_t)__shfl_sync(0xFFFFFFFFu, r, src);
        for (uint64_t j = lane; j < rk; j += 32) {
            out_probe[rb + j] = rr;
            out_build[rb + j] = T.rows[rs + j];
        }
    }
}

}  // namespace tplx
