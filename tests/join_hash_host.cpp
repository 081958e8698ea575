// Host shim over tuplex_b200/csrc/keyhash.cuh: the key hashes the CUDA join (join.cuh) calls, compiled for the CPU so that
// tests/test_join_edges.py can check its Python restatement of them. Test infrastructure only.
#include "../tuplex_b200/csrc/keyhash.cuh"
using namespace tplx;
extern "C" {
unsigned long long h_mix64(unsigned long long x) { return mix64(x); }
unsigned long long h_key_hash_i64(unsigned long long v) { return key_hash_i64(v); }
unsigned long long h_key_hash_bytes(const uint8_t *p, unsigned len) { return key_hash_bytes(p, len); }
}
