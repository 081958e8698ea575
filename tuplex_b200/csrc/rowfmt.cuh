// rowfmt.cuh — K5 row<->column transposition and K2 exception-row gather.
//
// The reference moves rows in its Tungsten-like row format inside fixed-size partitions
// (reference tuplex/utils/src/Serializer.cc:1016-1117, core/include/Partition.h:130-139):
//   row  = [one 8-byte slot per field][8 B total var-len bytes iff any var-len field][var-len payload]
//   slot = i64 | f64 bits | bool as i64 | (offset_from_slot_address & 0xFFFFFFFF) | (size_incl_NUL << 32)
//   partition = int64 numRows, then rows back to back.
// A schema with Option[T] fields prefixes each row with a bitmap of ceil(n_opt / 64) 8-byte words (Serializer.cc:1041-1059, see
// RowFmtCols). The reader accepts the three forms a None string field takes in the reference's rows:
//   "" of size 0, slot = offset | 0              (a None produced by a UDF, FlattenedTuple.cc:628; what write_row writes)
//   slot = 0 when the row has no var-len bytes   (Serializer.cc:313-338, 1071: slots are filled only when there are bytes)
//   the null cell's text, slot = offset | size   (the compiled CSV path, FlattenedTuple.cc:1255-1293, 798-835: "N/A\0" in the
//                                                 payload and in the var-len total)
// A None field's slot value is never used: it becomes "" (strings) or 0 (numbers) in the column block.
// Exception record = int64 rowNo, ecCode, opID, size, then the ORIGINAL input row
// (core/include/physical/IExceptionableTask.h:22-36).
#pragma once
#include <stdint.h>
#include "vm.cuh"
#include "../../include/tplx_gpu.h"

namespace tplx {

constexpr int RF_NT = 256;

// rows are packed back to back, so slots are NOT 8-byte aligned in general: byte-wise accessors
__device__ __forceinline__ uint64_t ld64u(const uint8_t *p) {
    uint64_t v = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) v |= (uint64_t)p[k] << (8 * k);
    return v;
}
__device__ __forceinline__ void st64u(uint8_t *p, uint64_t v) {
#pragma unroll
    for (int k = 0; k < 8; ++k) p[k] = (uint8_t)(v >> (8 * k));
}

// ---- generic exclusive scan over uint64 (three small kernels; boundary path, not the hot path) ---
constexpr int SCAN_ITEMS = 2048;  // per block
// The three kernels also run batched: blockIdx.y selects one of several arrays laid out `stride` elements apart (its
// block sums `sums_stride` apart), so K scans cost 3 launches instead of 3 K (used by the CSV source).
__global__ void scan_block_sums(const uint64_t *in, uint64_t *block_sums, uint64_t n, uint64_t stride = 0, uint64_t sums_stride = 0) {
    in += blockIdx.y * stride;
    block_sums += blockIdx.y * sums_stride;
    __shared__ uint64_t s[RF_NT / 32];
    uint64_t base = (uint64_t)blockIdx.x * SCAN_ITEMS;
    uint64_t v = 0;
    for (uint32_t i = threadIdx.x; i < SCAN_ITEMS; i += RF_NT)
        if (base + i < n) v += in[base + i];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t t = 0;
        for (int w = 0; w < RF_NT / 32; ++w) t += s[w];
        block_sums[blockIdx.x] = t;
    }
}
// single block: exclusive scan of block sums in place; total -> block_sums[n_blocks]
__global__ void scan_of_sums(uint64_t *block_sums, uint32_t n_blocks, uint64_t sums_stride = 0) {
    block_sums += blockIdx.y * sums_stride;
    __shared__ uint64_t s[1024 / 32];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t b0 = 0; b0 < n_blocks; b0 += 1024) {
        uint32_t i = b0 + threadIdx.x;
        uint64_t v = i < n_blocks ? block_sums[i] : 0, inc = v;
        for (int o = 1; o < 32; o <<= 1) {
            uint64_t a = __shfl_up_sync(0xFFFFFFFFu, inc, o);
            if ((threadIdx.x & 31) >= (uint32_t)o) inc += a;
        }
        if ((threadIdx.x & 31) == 31) s[threadIdx.x >> 5] = inc;
        __syncthreads();
        uint64_t wofs = 0;
        for (uint32_t w = 0; w < (threadIdx.x >> 5); ++w) wofs += s[w];
        uint64_t c = carry;
        if (i < n_blocks) block_sums[i] = c + wofs + inc - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + wofs + inc;
        __syncthreads();
    }
    if (threadIdx.x == 0) block_sums[n_blocks] = carry;
}
// out[i] = exclusive prefix (may alias in); out[n] = total when write_total
__global__ void scan_downsweep(const uint64_t *in, uint64_t *out, const uint64_t *block_sums, uint64_t n, int write_total,
                               uint64_t stride = 0, uint64_t sums_stride = 0) {
    in += blockIdx.y * stride;
    out += blockIdx.y * stride;
    block_sums += blockIdx.y * sums_stride;
    __shared__ uint64_t s[RF_NT / 32];
    const uint32_t per = SCAN_ITEMS / RF_NT;
    uint64_t base = (uint64_t)blockIdx.x * SCAN_ITEMS + (uint64_t)threadIdx.x * per;
    uint64_t vals[per];
    uint64_t mine = 0;
    for (uint32_t j = 0; j < per; ++j) {
        vals[j] = base + j < n ? in[base + j] : 0;
        mine += vals[j];
    }
    uint64_t inc = mine;
    for (int o = 1; o < 32; o <<= 1) {
        uint64_t a = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if ((threadIdx.x & 31) >= (uint32_t)o) inc += a;
    }
    if ((threadIdx.x & 31) == 31) s[threadIdx.x >> 5] = inc;
    __syncthreads();
    uint64_t wofs = 0;
    for (uint32_t w = 0; w < (threadIdx.x >> 5); ++w) wofs += s[w];
    uint64_t run = block_sums[blockIdx.x] + wofs + inc - mine;
    for (uint32_t j = 0; j < per; ++j) {
        if (base + j < n) out[base + j] = run;
        run += vals[j];
    }
    if (write_total && blockIdx.x == gridDim.x - 1 && threadIdx.x == RF_NT - 1) out[n] = block_sums[gridDim.x];
}

struct RowFmtCols {
    uint32_t n_cols, n_str;
    uint8_t types[TPLX_MAX_COLS];
    int8_t strk[TPLX_MAX_COLS];
    // column block side
    uint64_t *data[TPLX_MAX_COLS];      // fixed width values / (partitions->columns) destination
    uint32_t *offsets[TPLX_MAX_COLS];   // string offsets (n+1)
    uint8_t *bytes[TPLX_MAX_COLS];      // string bytes
    // Option[T] fields (Serializer.cc:1041-1059): the row starts with a bitmap of ceil(n_opt / 64) 8-byte words, bit k set = the k-th
    // Option field of the row is None; a None string field has size 0 and no bytes (appendWithoutInference(option<string>), :313-338)
    uint32_t n_opt, bitmap_bytes;
    int8_t optk[TPLX_MAX_COLS];         // index among the Option fields, -1 = not an Option field
    uint32_t *valid[TPLX_MAX_COLS];     // column block side: validity words (bit set = value present)
};

__device__ __forceinline__ bool rf_present(const RowFmtCols &C, uint32_t c, uint64_t i) {
    return C.optk[c] < 0 || !C.valid[c] || ((C.valid[c][i >> 5] >> (i & 31)) & 1u);
}

// ---- partitions -> columns ----------------------------------------------------------------------
// pass 1: fixed-width fields + string lengths (as uint64 for the scan)
__global__ void rows_to_cols_pass1(const uint8_t *__restrict__ rows, const uint64_t *__restrict__ row_off, uint64_t n,
                                   RowFmtCols C, uint64_t *__restrict__ lens /* [n_str][n+1] */) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i < n;
    const uint8_t *bm = active ? rows + row_off[i] : rows;
    const uint8_t *slots = bm + C.bitmap_bytes;
    for (uint32_t c = 0; c < C.n_cols; ++c) {
        bool isnull = false;
        if (C.optk[c] >= 0) {  // whole warps take this branch together: one validity word per warp and Option column
            if (active) isnull = (ld64u(bm + 8 * (size_t)(C.optk[c] >> 6)) >> (C.optk[c] & 63)) & 1ull;
            const uint32_t w = __ballot_sync(0xFFFFFFFFu, active && !isnull);
            if ((threadIdx.x & 31) == 0 && (i >> 5) < ((n + 31) >> 5)) C.valid[c][i >> 5] = w;
        }
        if (!active) continue;
        uint64_t v = ld64u(slots + 8 * (size_t)c);
        if (C.types[c] == TPLX_T_STR) lens[(size_t)C.strk[c] * (n + 1) + i] = (!isnull && (v >> 32)) ? (v >> 32) - 1 : 0;  // drop the NUL
        else C.data[c][i] = isnull ? 0 : v;
    }
}
// pass 2: string bytes (lens now holds exclusive byte offsets). The length is the one pass 1 counted, never the slot's: a None
// field may carry the null cell's text in its slot (the compiled CSV path), and pass 1 counted 0 bytes for it.
__global__ void rows_to_cols_pass2(const uint8_t *__restrict__ rows, const uint64_t *__restrict__ row_off, uint64_t n,
                                   RowFmtCols C, const uint64_t *__restrict__ lens) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    for (uint32_t c = 0; c < C.n_cols; ++c) {
        if (C.types[c] != TPLX_T_STR) continue;
        const uint64_t o = lens[(size_t)C.strk[c] * (n + 1) + i];
        C.offsets[c][i] = (uint32_t)o;
        if (i == n) continue;
        const uint32_t len = (uint32_t)(lens[(size_t)C.strk[c] * (n + 1) + i + 1] - o);
        if (!len) continue;  // "" or None: the slot is not read
        const uint8_t *slot = rows + row_off[i] + C.bitmap_bytes + 8 * (size_t)c;
        const uint8_t *src = slot + (uint32_t)ld64u(slot);
        uint8_t *dst = C.bytes[c] + o;
        for (uint32_t k = 0; k < len; ++k) dst[k] = src[k];
    }
}

// ---- columns -> rows ------------------------------------------------------------------------------
// serialized size of row i of a column block
__device__ __forceinline__ uint64_t row_size(const RowFmtCols &C, uint64_t i) {
    uint64_t sz = 8ull * C.n_cols + C.bitmap_bytes;
    if (C.n_str) {
        sz += 8;
        for (uint32_t c = 0; c < C.n_cols; ++c)
            if (C.types[c] == TPLX_T_STR && rf_present(C, c, i)) sz += (uint64_t)(C.offsets[c][i + 1] - C.offsets[c][i]) + 1;
    }
    return sz;
}
__device__ __forceinline__ void write_row(const RowFmtCols &C, uint64_t i, uint8_t *dst) {
    if (C.bitmap_bytes) {  // bit k = the k-th Option field is None
        for (uint32_t w = 0; w < C.bitmap_bytes / 8; ++w) {
            uint64_t bits = 0;
            for (uint32_t c = 0; c < C.n_cols; ++c)
                if (C.optk[c] >= 0 && (uint32_t)(C.optk[c] >> 6) == w && !rf_present(C, c, i)) bits |= 1ull << (C.optk[c] & 63);
            st64u(dst + 8 * (size_t)w, bits);
        }
        dst += C.bitmap_bytes;
    }
    uint64_t var = 8ull * C.n_cols + 8, total = 0;
    for (uint32_t c = 0; c < C.n_cols; ++c) {
        if (!rf_present(C, c, i)) {  // None: a zero slot; a string field still records where the next one starts, with size 0
            st64u(dst + 8 * (size_t)c, C.types[c] == TPLX_T_STR ? ((var - 8ull * c) & 0xFFFFFFFFull) : 0ull);
            continue;
        }
        if (C.types[c] == TPLX_T_STR) {
            const uint32_t o0 = C.offsets[c][i], len = C.offsets[c][i + 1] - o0;
            const uint64_t rel = var - 8ull * c;
            st64u(dst + 8 * (size_t)c, (rel & 0xFFFFFFFFull) | ((uint64_t)(len + 1) << 32));
            uint8_t *p = dst + var;
            const uint8_t *src = C.bytes[c] + o0;
            for (uint32_t k = 0; k < len; ++k) p[k] = src[k];
            p[len] = 0;
            var += len + 1;
            total += len + 1;
        } else st64u(dst + 8 * (size_t)c, C.data[c][i]);
    }
    if (C.n_str) st64u(dst + 8 * (size_t)C.n_cols, total);
}

__global__ void cols_row_sizes(RowFmtCols C, uint64_t n, uint64_t *sizes) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) sizes[i] = row_size(C, i);
}

// greedy partition split like rowToMemorySink (TransformTask.h:72-80): a row goes to a new partition when
// bytesWritten + size > capacity. row_off = exclusive prefix of sizes (n+1 entries). One thread; few partitions.
__global__ void split_partitions(const uint64_t *row_off, uint64_t n, uint64_t capacity, uint64_t *part_first_row,
                                 uint32_t max_parts, uint32_t *n_parts) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t np = 0;
    uint64_t start = 0;
    while (start < n && np < max_parts) {
        part_first_row[np++] = start;
        // largest e with row_off[e] - row_off[start] <= capacity  (at least one row per partition)
        uint64_t lo = start + 1, hi = n;
        while (lo < hi) {
            uint64_t mid = (lo + hi + 1) / 2;
            if (row_off[mid] - row_off[start] <= capacity) lo = mid; else hi = mid - 1;
        }
        start = lo;
    }
    if (n == 0 && max_parts) part_first_row[np++] = 0;  // one empty partition
    part_first_row[np] = n;
    *n_parts = (start < n) ? 0xFFFFFFFFu : np;
}

// rows -> partition buffer: partition p occupies [8*p + row_off[first_p], ...) + header
__global__ void cols_to_rows(RowFmtCols C, uint64_t n, const uint64_t *row_off, const uint64_t *part_first_row,
                             uint32_t n_parts, uint8_t *out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_parts) {
        uint64_t f = part_first_row[i], l = part_first_row[i + 1];
        st64u(out + 8ull * i + row_off[f], (uint64_t)(l - f));
    }
    if (i >= n) return;
    // find partition (few partitions: linear scan from the back is fine)
    uint32_t p = 0;
    while (p + 1 < n_parts && part_first_row[p + 1] <= i) ++p;
    write_row(C, i, out + 8ull * (p + 1) + row_off[i]);
}

// ---- K2: exception rows -------------------------------------------------------------------------
__global__ void exc_sizes(RowFmtCols Cin, const tplx_exception_rec *recs, uint64_t n_exc, uint64_t *sizes) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_exc) sizes[i] = 32 + row_size(Cin, (uint64_t)recs[i].row);
}
__global__ void exc_write(RowFmtCols Cin, const tplx_exception_rec *recs, uint64_t n_exc, const uint64_t *off, uint8_t *out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) st64u(out, n_exc);
    if (i >= n_exc) return;
    uint8_t *dst = out + 8 + off[i];
    const tplx_exception_rec r = recs[i];
    st64u(dst, (uint64_t)r.row_no);
    st64u(dst + 8, (uint64_t)r.code);
    st64u(dst + 16, (uint64_t)r.op_id);
    st64u(dst + 24, off[i + 1] - off[i] - 32);
    write_row(Cin, (uint64_t)r.row, dst + 32);
}

}  // namespace tplx
