// Host shim over tuplex_b200/csrc/keyhash.cuh: the key encodings of the device key sort (sort.cuh), compiled for the CPU so that
// tests/test_sort_keys.py can check that they order keys as Python does. Test infrastructure only.
#include "../tuplex_b200/csrc/keyhash.cuh"
using namespace tplx;
extern "C" {
unsigned long long h_sort_key_i64(long long v) { return sort_key_i64(v); }
unsigned long long h_sort_str_word(const uint8_t *p, unsigned len, unsigned k) { return sort_str_word(p, len, k); }
unsigned h_sort_str_class(unsigned len, unsigned k) { return sort_str_class(len, k); }
}
