// keyhash.cuh — the 64-bit key hashes of the hash tables (K4 hashagg.cuh, K8 join.cuh).
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

}  // namespace tplx
