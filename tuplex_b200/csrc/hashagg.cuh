// hashagg.cuh — K4 hash aggregate (aggregateByKey / unique).
//
// Replaces buildWithHashmapWriter + writeRowToHashTableAggregate + createFinalHashmap
// (reference tuplex/core/src/physical/PipelineBuilder.cc:1108-1400,
//  core/src/physical/TransformTask.cc:791-866, core/src/ee/local/LocalBackend.cc:2219-2376).
// The reference keeps one malloc'd bucket per key in a CityHash open-addressing map per task and
// merges the per-task maps on the driver. Here: ONE open-addressing table per (stage, device) in HBM,
// claimed with atomicCAS; key bytes live in a bump-allocated heap; per-CTA pre-aggregation buckets in
// shared memory absorb hot keys so that low-cardinality group-bys do not serialise on L2 atomics.
// Only the result SET must equal the reference's (SURVEY.md §2 row 12) — not the probing scheme.
#pragma once
#include <stdint.h>
#include "kernels.cuh"
#include "keyhash.cuh"

namespace tplx {

constexpr uint32_t HT_NOT_FOUND = 0xFFFFFFFFu;
constexpr uint32_t SM_BUCKETS = 1024;  // shared-memory pre-aggregation buckets per CTA
constexpr uint32_t SM_PROBES = 4;

struct HashTableDev {
    uint64_t *state;    // 0 empty, 1 busy, else fingerprint (hash | 2)
    uint64_t *keyoff;   // heap offset | blob size << 40
    uint64_t *accs;     // [n_accs][cap]
    uint8_t *heap;      // key blobs: per key column i64 -> 8 bytes, str -> u32 len + bytes; an Option key column puts one flag
                        // byte in front (1 = None, and then nothing follows; 0 = the value's encoding follows)
    uint64_t cap, mask, max_keys, heap_cap;
    uint64_t *counters; // [0] n_keys, [1] heap_used, [2] overflow rows, [3] exception append
};

struct HashTable {
    HashTableDev d{};
    int device = -1;
    uint32_t n_accs = 0;
};

struct HashParams {
    HashTableDev ht;
    uint32_t n_keys;
    uint32_t key_slot[TPLX_MAX_KEYS];
    uint32_t key_type[TPLX_MAX_KEYS];
    uint32_t key_null[TPLX_MAX_KEYS];  // slot of key k's "is None" flag, TPLX_NOSLOT when key k cannot be None
    const uint32_t *rowlist;   // optional: process these rows only (overflow retry)
    uint64_t n_list;
    uint32_t *overflow_rows;   // rows whose key could not be inserted (table/heap full)
    uint64_t cap_overflow;
};

// A None key is one group whatever its value slot holds (the other branch of a select, junk under an invalid input row): the slot
// is never read for it, so it reaches neither the hash nor the comparison nor the blob. OPT: the stage has Option keys (a stage
// without them runs code in which none of these tests exist).
template <int NTT>
__device__ __forceinline__ bool key_is_none(const HashParams &H, uint8_t *regs, uint32_t k) {
    return H.key_null[k] != TPLX_NOSLOT && VM<NTT>::R(regs, H.key_null[k] * VM<NTT>::SLOT_BYTES) != 0;
}

template <int NTT, bool OPT>
__device__ __forceinline__ uint64_t hash_key(const HashParams &H, uint8_t *regs, uint32_t *blob_size) {
    uint64_t h = 0x9E3779B97F4A7C15ull;
    uint32_t sz = 0;
    for (uint32_t k = 0; k < H.n_keys; ++k) {
        if (OPT && H.key_null[k] != TPLX_NOSLOT) {
            sz += 1;
            if (key_is_none<NTT>(H, regs, k)) {
                h = mix64(h ^ 0x4E6F6E654B657921ull);
                continue;
            }
        }
        if (H.key_type[k] == TPLX_T_STR) {
            StrV s = VM<NTT>::RS(regs, H.key_slot[k] * VM<NTT>::SLOT_BYTES);
            uint64_t f = 0xcbf29ce484222325ull;
            for (uint32_t i = 0; i < s.len; ++i) f = (f ^ sch(s, i)) * 0x100000001b3ull;
            h = mix64(h ^ f ^ ((uint64_t)s.len << 48));
            sz += 4 + s.len;
        } else {
            h = mix64(h ^ VM<NTT>::R(regs, H.key_slot[k] * VM<NTT>::SLOT_BYTES));
            sz += 8;
        }
    }
    *blob_size = sz;
    return h;
}

template <int NTT, bool OPT>
__device__ __forceinline__ bool key_equal(const HashParams &H, uint8_t *regs, const uint8_t *blob) {
    for (uint32_t k = 0; k < H.n_keys; ++k) {
        if (OPT && H.key_null[k] != TPLX_NOSLOT) {
            const bool none = key_is_none<NTT>(H, regs, k);
            if ((*blob++ != 0) != none) return false;
            if (none) continue;
        }
        if (H.key_type[k] == TPLX_T_STR) {
            StrV s = VM<NTT>::RS(regs, H.key_slot[k] * VM<NTT>::SLOT_BYTES);
            uint32_t len = blob[0] | (blob[1] << 8) | (blob[2] << 16) | ((uint32_t)blob[3] << 24);
            if (len != s.len) return false;
            blob += 4;
            for (uint32_t i = 0; i < len; ++i)
                if (blob[i] != sch(s, i)) return false;
            blob += len;
        } else {
            uint64_t v = 0;
            for (int b = 0; b < 8; ++b) v |= (uint64_t)blob[b] << (8 * b);
            if (v != VM<NTT>::R(regs, H.key_slot[k] * VM<NTT>::SLOT_BYTES)) return false;
            blob += 8;
        }
    }
    return true;
}

template <int NTT, bool OPT>
__device__ __forceinline__ void key_write(const HashParams &H, uint8_t *regs, uint8_t *blob) {
    for (uint32_t k = 0; k < H.n_keys; ++k) {
        if (OPT && H.key_null[k] != TPLX_NOSLOT) {
            const bool none = key_is_none<NTT>(H, regs, k);
            *blob++ = none ? 1 : 0;
            if (none) continue;
        }
        if (H.key_type[k] == TPLX_T_STR) {
            StrV s = VM<NTT>::RS(regs, H.key_slot[k] * VM<NTT>::SLOT_BYTES);
            blob[0] = (uint8_t)s.len; blob[1] = (uint8_t)(s.len >> 8); blob[2] = (uint8_t)(s.len >> 16); blob[3] = (uint8_t)(s.len >> 24);
            blob += 4;
            str_copy(blob, s);
            blob += s.len;
        } else {
            uint64_t v = VM<NTT>::R(regs, H.key_slot[k] * VM<NTT>::SLOT_BYTES);
            for (int b = 0; b < 8; ++b) blob[b] = (uint8_t)(v >> (8 * b));
            blob += 8;
        }
    }
}

__device__ __forceinline__ uint64_t ld_acquire_u64(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u64(uint64_t *p, uint64_t v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// returns table slot of the key, inserting it if absent; HT_NOT_FOUND when the table or heap is full
template <int NTT, bool OPT>
__device__ uint32_t find_or_insert(const HashParams &H, uint8_t *regs, uint64_t h, uint32_t blob_size) {
    const HashTableDev &T = H.ht;
    const uint64_t fp = h | 2ull;
    uint64_t idx = (h >> 17) & T.mask;
    for (uint64_t probe = 0; probe <= T.mask; ++probe) {
        uint64_t st = ld_cg_u64(&T.state[idx]);
        while (true) {
            if (st == 0) {
                if (ld_cg_u64(&T.counters[0]) >= T.max_keys) return HT_NOT_FOUND;
                uint64_t prev = atomicCAS((unsigned long long *)&T.state[idx], 0ull, 1ull);
                if (prev == 0) {
                    uint64_t nk = atomicAdd((unsigned long long *)&T.counters[0], 1ull);
                    uint64_t off = 0;
                    bool ok = nk < T.max_keys;
                    if (ok) {
                        off = atomicAdd((unsigned long long *)&T.counters[1], (unsigned long long)blob_size);
                        ok = off + blob_size <= T.heap_cap;
                    }
                    if (!ok) {
                        atomicAdd((unsigned long long *)&T.counters[0], (unsigned long long)-1ll);
                        st_release_u64(&T.state[idx], 0ull);
                        return HT_NOT_FOUND;
                    }
                    key_write<NTT, OPT>(H, regs, T.heap + off);
                    T.keyoff[idx] = off | ((uint64_t)blob_size << 40);
                    __threadfence();
                    st_release_u64(&T.state[idx], fp);
                    return (uint32_t)idx;
                }
                st = prev;
            }
            if (st == 1) { st = ld_acquire_u64(&T.state[idx]); continue; }
            break;
        }
        if (st == fp) {
            __threadfence();
            const uint64_t ko = ld_cg_u64(&T.keyoff[idx]);
            if ((uint32_t)(ko >> 40) == blob_size && key_equal<NTT, OPT>(H, regs, T.heap + (ko & ((1ull << 40) - 1)))) return (uint32_t)idx;
        }
        idx = (idx + 1) & T.mask;
    }
    return HT_NOT_FOUND;
}

__device__ __forceinline__ void atomic_acc_global(uint32_t kind, uint64_t *p, uint64_t v) {
    switch (kind) {
        case TPLX_ACC_SUM_I64: atomicAdd((unsigned long long *)p, (unsigned long long)v); break;
        case TPLX_ACC_SUM_F64: atomicAdd((double *)p, __longlong_as_double((long long)v)); break;
        case TPLX_ACC_MIN_I64: atomicMin((long long *)p, (long long)v); break;
        case TPLX_ACC_MAX_I64: atomicMax((long long *)p, (long long)v); break;
        default: {
            unsigned long long old = *(volatile unsigned long long *)p;
            while (true) {
                uint64_t nv = acc_combine(kind, old, v);
                if (nv == old) break;
                unsigned long long prev = atomicCAS((unsigned long long *)p, old, nv);
                if (prev == old) break;
                old = prev;
            }
        }
    }
}

#ifndef TPLX_JIT
// fill accumulator arrays with identities
__global__ void hash_init_accs(HashTableDev T, uint32_t n_accs, const AccP *accs_dev_unused, uint32_t k0, uint32_t kind) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < T.cap) T.accs[(size_t)k0 * T.cap + i] = acc_identity(kind);
}

// =============================================================================================
// K4: rows in -> hash table.  Same tile/VM structure as K3; the per-row sink is the table.
// EXC_ONLY: collect the exception records only and leave the table alone (second pass over a block whose exception rows did
// not fit the first pass's buffer). OPT_KEYS: some key column can be None (HashParams.key_null).
// =============================================================================================
template <bool EXC_ONLY, bool OPT_KEYS>
__global__ void __launch_bounds__(NT) stage_hash_kernel(const KParams *__restrict__ Pg, const HashParams *__restrict__ Hg) {
    extern __shared__ __align__(16) uint8_t smem[];
    const KParams &P = *Pg;
    const HashParams &H = *Hg;
    const uint32_t tid = threadIdx.x;
    const uint32_t R = P.R, T = R * NT;

    DInstr *s_prog = reinterpret_cast<DInstr *>(smem);
    ColIn *s_cols = reinterpret_cast<ColIn *>(smem + P.smem_cols_off);
    uint8_t *s_regs = smem + P.smem_regs_off + tid * 8;  // this thread's register column
    // pre-aggregation buckets: gidx[SM_BUCKETS] (u32) then acc[n_accs][SM_BUCKETS] (u64)
    uint64_t *s_bacc = reinterpret_cast<uint64_t *>(smem + P.smem_misc_off);
    uint32_t *s_bkey = reinterpret_cast<uint32_t *>(s_bacc + (size_t)P.n_accs * SM_BUCKETS);
    uint32_t *s_stat = s_bkey + SM_BUCKETS;  // [0] bucket hits, [1] bucket misses, [2] disabled

    for (uint32_t i = tid; i < P.n_instr * (sizeof(DInstr) / 16); i += NT)
        reinterpret_cast<uint4 *>(s_prog)[i] = reinterpret_cast<const uint4 *>(P.prog)[i];
    for (uint32_t i = tid; i < P.n_in * (sizeof(ColIn) / 8); i += NT)
        reinterpret_cast<uint64_t *>(s_cols)[i] = reinterpret_cast<const uint64_t *>(P.in)[i];
    if (!EXC_ONLY)
        for (uint32_t i = tid; i < SM_BUCKETS; i += NT) {
            s_bkey[i] = HT_NOT_FOUND;
            for (uint32_t k = 0; k < P.n_accs; ++k) s_bacc[(size_t)k * SM_BUCKETS + i] = acc_identity(P.accs[k].kind);
        }
    if (tid < 4) s_stat[tid] = 0;
    __syncthreads();

    VMThread t;
    t.scr_cap = P.scratch_per_thread;
    t.scratch = P.scratch + ((size_t)blockIdx.x * NT + tid) * (size_t)P.scratch_per_thread;
    const uint32_t na = P.n_accs;
    const uint64_t n_work = H.rowlist ? H.n_list : P.n_rows;
    const uint32_t n_tiles = (uint32_t)((n_work + T - 1) / T);

    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint64_t base = (uint64_t)tile * T;
        for (uint32_t s = 0; s < R; ++s) {
            const uint64_t w = base + (uint64_t)s * NT + tid;
            const bool valid = w < n_work;
            const uint64_t row = valid ? (H.rowlist ? (uint64_t)H.rowlist[w] : w) : 0;
            t.alive = valid;
            t.exc_code = 0;
            t.scr_used = 0;
            VM<NT>::run(s_prog, 0, P.n_instr, s_regs, s_cols, row, row, P.cpool, t);
            if (!EXC_ONLY && t.alive) {
                uint32_t blob = 0;
                const uint64_t h = hash_key<NT, OPT_KEYS>(H, s_regs, &blob);
                const uint32_t g = find_or_insert<NT, OPT_KEYS>(H, s_regs, h, blob);
                if (g == HT_NOT_FOUND) {
                    uint64_t pos = atomicAdd((unsigned long long *)&H.ht.counters[2], 1ull);
                    if (pos < H.cap_overflow) H.overflow_rows[pos] = (uint32_t)row;
                } else if (na) {
                    // shared-memory pre-aggregation bucket keyed by the (exact) table slot
                    bool done = false;
                    if (!s_stat[2]) {
                        uint32_t b = (g * 2654435761u) >> 22;  // 10 bits
                        for (uint32_t pr = 0; pr < SM_PROBES && !done; ++pr) {
                            uint32_t prev = atomicCAS(&s_bkey[b], HT_NOT_FOUND, g);
                            if (prev == HT_NOT_FOUND || prev == g) {
                                for (uint32_t k = 0; k < na; ++k) {
                                    uint64_t v = VM<NT>::R(s_regs, P.accs[k].slot * VM<NT>::SLOT_BYTES);
                                    uint64_t *p = &s_bacc[(size_t)k * SM_BUCKETS + b];
                                    switch (P.accs[k].kind) {
                                        case TPLX_ACC_SUM_I64: atomicAdd((unsigned long long *)p, (unsigned long long)v); break;
                                        case TPLX_ACC_SUM_F64: atomicAdd((double *)p, __longlong_as_double((long long)v)); break;
                                        case TPLX_ACC_MIN_I64: atomicMin((long long *)p, (long long)v); break;
                                        case TPLX_ACC_MAX_I64: atomicMax((long long *)p, (long long)v); break;
                                        default: {
                                            unsigned long long old = *(volatile unsigned long long *)p;
                                            while (true) {
                                                uint64_t nv = acc_combine(P.accs[k].kind, old, v);
                                                if (nv == old) break;
                                                unsigned long long q = atomicCAS((unsigned long long *)p, old, nv);
                                                if (q == old) break;
                                                old = q;
                                            }
                                        }
                                    }
                                }
                                done = true;
                            }
                            b = (b + 1) & (SM_BUCKETS - 1);
                        }
                        atomicAdd(&s_stat[done ? 0 : 1], 1u);
                    }
                    if (!done)
                        for (uint32_t k = 0; k < na; ++k)
                            atomic_acc_global(P.accs[k].kind, &H.ht.accs[(size_t)k * H.ht.cap + g], VM<NT>::R(s_regs, P.accs[k].slot * VM<NT>::SLOT_BYTES));
                }
            }
            if (t.exc_code) {
                uint64_t pos = atomicAdd((unsigned long long *)&H.ht.counters[3], 1ull);
                if (pos < P.cap_exc) {
                    tplx_exception_rec rec;
                    rec.row = (int64_t)row;
                    rec.row_no = 0;
                    rec.code = t.exc_code;
                    rec.op_id = P.opids[t.exc_op];
                    P.exc[pos] = rec;
                } else atomicOr(&P.counters[1], 4u);
            }
        }
        __syncthreads();
        // high-cardinality input: buckets thrash -> stop using them (they are still flushed at the end)
        if (tid == 0 && !s_stat[2] && s_stat[1] > 4 * s_stat[0] + 1024) s_stat[2] = 1;
        __syncthreads();
    }
    // flush the pre-aggregation buckets
    if (!EXC_ONLY)
        for (uint32_t i = tid; i < SM_BUCKETS; i += NT) {
            const uint32_t g = s_bkey[i];
            if (g == HT_NOT_FOUND) continue;
            for (uint32_t k = 0; k < na; ++k)
                atomic_acc_global(P.accs[k].kind, &H.ht.accs[(size_t)k * H.ht.cap + g], s_bacc[(size_t)k * SM_BUCKETS + i]);
        }
}

// ---- table maintenance ----------------------------------------------------------------------------
// re-insert every entry of `old` into `neu` (growth); heap is shared (same offsets)
__global__ void hash_rehash(HashTableDev old, HashTableDev neu, uint32_t n_accs, const uint32_t *kinds) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= old.cap) return;
    const uint64_t st = old.state[i];
    if (st < 2) return;
    // fingerprint keeps all hash bits except bit 1, which does not take part in slot selection
    uint64_t idx = (st >> 17) & neu.mask;
    while (true) {
        uint64_t prev = atomicCAS((unsigned long long *)&neu.state[idx], 0ull, (unsigned long long)st);
        if (prev == 0) break;
        idx = (idx + 1) & neu.mask;
    }
    neu.keyoff[idx] = old.keyoff[i];
    for (uint32_t k = 0; k < n_accs; ++k) neu.accs[(size_t)k * neu.cap + idx] = old.accs[(size_t)k * old.cap + i];
}

// Owner rank of a key in the multi-GPU exchange: a function of the key's hash only (state = hash | 2), so every rank
// computes the same owner for equal keys. The high bits are independent of the bits that pick the table slot.
struct HashSel {
    int32_t owner;   // -1: every occupied slot, else only slots whose key is owned by this rank
    uint32_t world;
};
__device__ __forceinline__ bool slot_selected(uint64_t st, HashSel sel) {
    return st >= 2 && (sel.owner < 0 || (uint32_t)((st >> 40) % sel.world) == (uint32_t)sel.owner);
}
// finish: flag selected slots (uint64 0/1 for the scan) ...
__global__ void hash_flag_slots(HashTableDev T, uint64_t *flags, HashSel sel) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < T.cap) flags[i] = slot_selected(T.state[i], sel) ? 1 : 0;
}
struct HashEmit {
    uint32_t n_keys, n_accs;
    uint32_t key_types[TPLX_MAX_KEYS];
    uint32_t acc_kinds[TPLX_MAX_ACCS];
    int64_t acc_init[TPLX_MAX_ACCS];
    uint64_t *key_none[TPLX_MAX_KEYS];     // Option key columns: 1 where the group's key is None (packed into the validity bitmap
                                           // afterwards); nullptr for a key column that cannot be None
    uint64_t *key_data[TPLX_MAX_KEYS];     // i64 keys
    uint32_t *key_offsets[TPLX_MAX_KEYS];  // str keys: offsets (n+1)
    const uint64_t *key_lens_scan[TPLX_MAX_KEYS];  // exclusive byte offsets per compacted key (n+1)
    uint8_t *key_bytes[TPLX_MAX_KEYS];
    uint64_t *acc_data[TPLX_MAX_ACCS];
};
__device__ __forceinline__ uint32_t blob_u32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
// steps over the flag byte of an Option key column; true when the key is None (no value follows)
__device__ __forceinline__ bool blob_none(const uint8_t *&blob, const HashEmit &E, uint32_t k) {
    return E.key_none[k] && *blob++ != 0;
}
// ... per-key string lengths of key column kc at compacted position (for the per-column offset scan; 0 for a None key)
__global__ void hash_key_lens(HashTableDev T, const uint64_t *pos, HashEmit E, uint32_t kc, uint64_t *lens, HashSel sel) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T.cap || !slot_selected(T.state[i], sel)) return;
    const uint8_t *blob = T.heap + (T.keyoff[i] & ((1ull << 40) - 1));
    for (uint32_t k = 0; k < kc; ++k) {
        if (blob_none(blob, E, k)) continue;
        blob += E.key_types[k] == TPLX_T_STR ? 4 + blob_u32(blob) : 8;
    }
    lens[pos[i]] = blob_none(blob, E, kc) ? 0 : blob_u32(blob);
}
// ... and emit key + accumulator columns at the compacted position; a None key gets the placeholder value (0, empty string)
__global__ void hash_emit(HashTableDev T, const uint64_t *pos, uint64_t n_out, HashEmit E, HashSel sel) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0)
        for (uint32_t k = 0; k < E.n_keys; ++k)
            if (E.key_types[k] == TPLX_T_STR) E.key_offsets[k][n_out] = (uint32_t)E.key_lens_scan[k][n_out];
    if (i >= T.cap || !slot_selected(T.state[i], sel)) return;
    const uint64_t o = pos[i];
    const uint8_t *blob = T.heap + (T.keyoff[i] & ((1ull << 40) - 1));
    for (uint32_t k = 0; k < E.n_keys; ++k) {
        const bool none = blob_none(blob, E, k);
        if (E.key_none[k]) E.key_none[k][o] = none ? 1 : 0;
        if (none) {
            if (E.key_types[k] == TPLX_T_STR) E.key_offsets[k][o] = (uint32_t)E.key_lens_scan[k][o];
            else E.key_data[k][o] = 0;
            continue;
        }
        if (E.key_types[k] == TPLX_T_STR) {
            uint32_t len = blob[0] | (blob[1] << 8) | (blob[2] << 16) | ((uint32_t)blob[3] << 24);
            blob += 4;
            const uint64_t bo = E.key_lens_scan[k][o];
            E.key_offsets[k][o] = (uint32_t)bo;
            uint8_t *dst = E.key_bytes[k] + bo;
            for (uint32_t b = 0; b < len; ++b) dst[b] = blob[b];
            blob += len;
        } else {
            uint64_t v = 0;
            for (int b = 0; b < 8; ++b) v |= (uint64_t)blob[b] << (8 * b);
            E.key_data[k][o] = v;
            blob += 8;
        }
    }
    // bucket starts from the initial value, and combine(init, value) runs once per group at the end
    // (TransformTask.cc:358-375, LocalBackend.cc:2148-2217)
    for (uint32_t k = 0; k < E.n_accs; ++k) {
        uint64_t v = acc_combine(E.acc_kinds[k], (uint64_t)E.acc_init[k], T.accs[(size_t)k * T.cap + i]);
        v = acc_combine(E.acc_kinds[k], (uint64_t)E.acc_init[k], v);
        E.acc_data[k][o] = v;
    }
}

// merge packed rows (keys + partial accumulators already containing no init) from another table
// is done by running stage_hash_kernel with an identity program over the packed block (host side).

static inline void hash_table_destroy(HashTable *t) {
    if (!t) return;
    cudaSetDevice(t->device);
    cudaFree(t->d.state);
    cudaFree(t->d.keyoff);
    cudaFree(t->d.accs);
    cudaFree(t->d.heap);
    cudaFree(t->d.counters);
    delete t;
}

#endif  // !TPLX_JIT

}  // namespace tplx
