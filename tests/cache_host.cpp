// Host shim over tuplex_b200/csrc/cache.cuh: the UTF-8 rewrite of a cached string column with plain loops standing in for the
// grid — per-row length after the replacement, exclusive scan, per-row write — and the per-row validity test the block
// statistics count. tests/test_cache_plan.py compares it with CPython. Test infrastructure only.
#include "../tuplex_b200/csrc/cache.cuh"
#include <vector>
using namespace tplx;

extern "C" {
// rewrites the n strings of (bytes, offsets); returns the output bytes; out_offsets gets n + 1 entries, out_bytes (may be null)
// the bytes; *n_invalid = strings that change
uint64_t hcache_rewrite(const uint8_t *bytes, const uint32_t *offsets, uint64_t n, uint32_t *out_offsets, uint8_t *out_bytes,
                        uint64_t *n_invalid) {
    std::vector<uint64_t> pos(n + 1, 0);
    uint64_t bad = 0;
    for (uint64_t i = 0; i < n; ++i) {
        pos[i + 1] = pos[i] + cache_utf8_len(bytes, offsets, i);
        bad += cache_utf8_invalid(bytes, offsets, i) ? 1 : 0;
    }
    for (uint64_t i = 0; i <= n; ++i) out_offsets[i] = (uint32_t)pos[i];
    if (out_bytes)
        for (uint64_t i = 0; i < n; ++i) cache_utf8_write(bytes, offsets, i, out_bytes + pos[i]);
    *n_invalid = bad;
    return pos[n];
}
}
