// keyhash.cuh — the 64-bit key hashes of the hash tables (K4 hashagg.cuh, K8 join.cuh), and the order-preserving key encodings of
// the device key sort (K11 sort.cuh).
//
// mix64 is the MurmurHash3 fmix64 finaliser. The join hashes one key column with it: an i64 (or bool) key as mix64(v ^ golden
// ratio), a string key as FNV-1a over its bytes with the length folded into the high bits before mix64. The header compiles for
// the host too (TPLX_HD) so that tests/test_join_edges.py can check a Python restatement of these exact functions and build keys
// that share a probe chain on purpose.
#pragma once
#include <stdint.h>
#include "strops.cuh"

namespace tplx {

TPLX_HD uint64_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}

TPLX_HD uint64_t key_hash_i64(uint64_t v) { return mix64(v ^ 0x9E3779B97F4A7C15ull); }

TPLX_HD uint64_t key_hash_bytes(const uint8_t *p, uint32_t len) {
    uint64_t f = 0xcbf29ce484222325ull;
    for (uint32_t i = 0; i < len; ++i) f = (f ^ p[i]) * 0x100000001b3ull;
    return mix64(f ^ ((uint64_t)len << 48));
}

// ---- order-preserving key encodings of the device key sort (sort.cuh); tests/test_sort_keys.py checks them against Python ----
// i64: the sign bit flipped, so that unsigned order is signed order.
TPLX_HD uint64_t sort_key_i64(int64_t v) { return (uint64_t)v ^ 0x8000000000000000ull; }

// str: word k is the big-endian bytes [8k, 8k + 8), zero past the end; class k is min(len - 8k, 9), 0 past the end. Comparing
// (word_0, class_0), (word_1, class_1), ... lexicographically, word before class, up to the first pair whose class is below 9 is
// bytes order: a zero pad byte ties with a real NUL, and the class then puts the shorter string (a prefix of the other) first.
TPLX_HD uint64_t sort_str_word(const uint8_t *p, uint32_t len, uint32_t k) {
    const uint64_t b = (uint64_t)k * 8;
    uint64_t w = 0;
    for (uint32_t i = 0; i < 8; ++i) w = (w << 8) | (b + i < len ? p[b + i] : 0u);
    return w;
}

TPLX_HD uint32_t sort_str_class(uint32_t len, uint32_t k) {
    const uint64_t b = (uint64_t)k * 8;
    return b >= len ? 0u : (len - b >= 9 ? 9u : (uint32_t)(len - b));
}

}  // namespace tplx
