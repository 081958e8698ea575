// strops.cuh — string primitives of the VM, written word-at-a-time (SWAR over aligned 32-bit loads).
//
// Semantics restated from the reference (paths relative to /root/reference/tuplex/):
//   find    = strstr                       codegen/src/FunctionRegistry.cc:2165-2188
//   rfind   = std::string::rfind           runtime/src/Runtime.cc:387-397
//   ==      = strcmp == 0                  codegen/src/BlockGeneratorVisitor.cc:838-856
//   lower / upper: ASCII only, C locale    runtime/src/StringFunctions.cc:71-110
// A string value is a view (pointer, length, lazy case flag); see include/tplx_ir.h.
//
// Memory contract: a view's bytes live in a buffer whose allocation is a multiple of 4 bytes and 4-byte
// aligned at its base (all buffers this library allocates are), so every ALIGNED 32-bit word that contains
// at least one byte of the string may be loaded. Words that contain no string byte are never touched.
//
// The header compiles for the host too (TPLX_HD) so that tests/test_strops_host.py can fuzz these exact
// functions on the CPU against CPython's str methods.
#pragma once
#include <stdint.h>
#include "../../include/tplx_ir.h"

#ifdef __CUDACC__
#define TPLX_HD __host__ __device__ __forceinline__
#define TPLX_HD_NOINLINE __host__ __device__ __noinline__
#else
#define TPLX_HD inline
#define TPLX_HD_NOINLINE inline
#endif

namespace tplx {

struct StrV {
    const uint8_t *p;
    uint32_t len;
    uint32_t flags;
};

TPLX_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) {
#ifdef __CUDA_ARCH__
    return __funnelshift_r(lo, hi, sh);
#else
    return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}

// packed ASCII case mapping of 4 bytes; bytes >= 0x80 are left alone (tolower/toupper in the C locale)
TPLX_HD uint32_t lower4(uint32_t w) {
    uint32_t w7 = w & 0x7f7f7f7fu;
    uint32_t m = (w7 + 0x3f3f3f3fu) & ~(w7 + 0x25252525u) & ~w & 0x80808080u;  // 'A'..'Z'
    return w | (m >> 2);
}
TPLX_HD uint32_t upper4(uint32_t w) {
    uint32_t w7 = w & 0x7f7f7f7fu;
    uint32_t m = (w7 + 0x1f1f1f1fu) & ~(w7 + 0x05050505u) & ~w & 0x80808080u;  // 'a'..'z'
    return w & ~(m >> 2);
}
TPLX_HD uint32_t case4(uint32_t w, uint32_t flags) {
    return flags == TPLX_SF_LOWER ? lower4(w) : (flags == TPLX_SF_UPPER ? upper4(w) : w);
}
TPLX_HD uint8_t case1(uint8_t c, uint32_t flags) {  // branch-free (selects): it sits in the inner loops of byte-wise fallbacks
    const uint8_t lo = (flags == TPLX_SF_LOWER && (uint8_t)(c - 'A') < 26u) ? 32 : 0;
    const uint8_t up = (flags == TPLX_SF_UPPER && (uint8_t)(c - 'a') < 26u) ? 32 : 0;
    return (uint8_t)(c + lo - up);
}
// 0x80 in every byte lane of w that equals c (exact, no false positives)
TPLX_HD uint32_t eq_mask4(uint32_t w, uint32_t c) {
    uint32_t x = w ^ (c * 0x01010101u);
    uint32_t t = ((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x;
    return ~t & 0x80808080u;
}

TPLX_HD uint8_t sch(const StrV &s, uint32_t i) { return case1(s.p[i], s.flags); }

// Sequential reader of a string as little-endian 32-bit words of 4 characters (word k = chars 4k..4k+3),
// built from aligned loads + funnel shift. Characters past the end read as garbage: callers mask.
struct WordReader {
    const uint32_t *w;  // aligned base
    uint32_t sh;        // bit offset of the string start inside *w
    uint32_t nwords;    // aligned words that contain string bytes
    uint32_t flags;
    TPLX_HD void init(const StrV &s) {
        uintptr_t a = (uintptr_t)s.p;
        w = (const uint32_t *)(a & ~(uintptr_t)3);
        sh = (uint32_t)(a & 3) * 8;
        nwords = (uint32_t)(((a & 3) + s.len + 3) >> 2);
        flags = s.flags;
    }
    TPLX_HD uint32_t aligned(uint32_t j) const { return j < nwords ? w[j] : 0u; }
    // characters 4k..4k+3 (case-mapped)
    TPLX_HD uint32_t get(uint32_t k) const {
        uint32_t lo = aligned(k);
        uint32_t hi = sh ? aligned(k + 1) : 0u;
        return case4(funnel_r(lo, hi, sh), flags);
    }
};

TPLX_HD uint32_t low_mask(uint32_t nbytes) {  // mask of the low nbytes (0..4) bytes
    return nbytes >= 4 ? 0xFFFFFFFFu : ((1u << (8 * nbytes)) - 1u);
}

// Copy the (case-mapped) characters of s to dst, four at a time: dst is written with aligned 32-bit stores between an unaligned head
// and tail (bytes that share a word with a neighbouring string are only ever written as bytes), src is read with aligned loads and a
// funnel shift (memory contract above). Replaces `for i: dst[i] = sch(s, i)`: ~8 instructions per 4 characters instead of ~12 per character.
TPLX_HD void str_copy(uint8_t *dst, const StrV &s) {
    const uint32_t n = s.len;
    uint32_t i = 0;
    while (i < n && ((uintptr_t)(dst + i) & 3)) {
        dst[i] = sch(s, i);
        ++i;
    }
    if (i + 4 <= n) {
        const uintptr_t a = (uintptr_t)(s.p + i);
        const uint32_t *aw = (const uint32_t *)(a & ~(uintptr_t)3);
        const uint32_t sh = (uint32_t)(a & 3) * 8;
        uint32_t *dw = (uint32_t *)(dst + i);
        if (sh == 0) {
            for (; i + 4 <= n; i += 4) *dw++ = case4(*aw++, s.flags);
        } else {
            uint32_t cur = *aw++;
            for (; i + 4 <= n; i += 4) {  // characters i..i+3 straddle two aligned words, both hold string bytes
                const uint32_t nxt = *aw++;
                *dw++ = case4(funnel_r(cur, nxt, sh), s.flags);
                cur = nxt;
            }
        }
    }
    for (; i < n; ++i) dst[i] = sch(s, i);
}

// The out-of-line primitives (here and in vm.cuh) take their views by value: a reference parameter makes every call store the
// caller's StrV to the thread's stack and the callee load it back, local-memory traffic on every string op of a row function.
// a == b (both possibly case-flagged)
TPLX_HD_NOINLINE bool str_eq(StrV a, StrV b) {
    if (a.len != b.len) return false;
    WordReader ra, rb;
    ra.init(a);
    rb.init(b);
    const uint32_t n = a.len;
    for (uint32_t k = 0; 4 * k < n; ++k) {
        uint32_t x = ra.get(k) ^ rb.get(k);
        uint32_t rem = n - 4 * k;
        if (x & low_mask(rem)) return false;
    }
    return true;
}

// does hay[pos..pos+n.len) equal n ? (byte path, used to verify SWAR candidates)
TPLX_HD bool match_at(const StrV &h, uint32_t pos, const StrV &n, uint32_t from) {
    for (uint32_t j = from; j < n.len; ++j)
        if (sch(h, pos + j) != sch(n, j)) return false;
    return true;
}

// 0x80 in every byte lane where BOTH x0 and x1 are zero (x0, x1 = word ^ splat(char)): one zero-byte test for a 2-character filter
TPLX_HD uint32_t both_zero4(uint32_t x0, uint32_t x1) {
    const uint32_t x = x0 | x1;
    const uint32_t t = ((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x;
    return ~t & 0x80808080u;
}
template <uint32_t HFLAGS>
TPLX_HD uint32_t case4_t(uint32_t w) {
    return HFLAGS == TPLX_SF_LOWER ? lower4(w) : (HFLAGS == TPLX_SF_UPPER ? upper4(w) : w);
}
template <uint32_t HFLAGS>
TPLX_HD uint8_t sch_t(const uint8_t *p, uint32_t i) {
    uint8_t c = p[i];
    if (HFLAGS == TPLX_SF_LOWER) c += ((uint8_t)(c - 'A') < 26u) ? 32 : 0;
    if (HFLAGS == TPLX_SF_UPPER) c -= ((uint8_t)(c - 'a') < 26u) ? 32 : 0;
    return c;
}

// strstr semantics: first occurrence or -1 (callers handle the empty needle and needle longer than haystack).
// SWAR filter on the first (and, when present, second) needle character, 4 haystack positions per step. One aligned load per step:
// string word k (characters 4k..4k+3) = funnel(aw[k], aw[k+1]); the character after it — needed for the 2-character test of position
// 4k+3 — is the byte at the string's phase inside aw[k+1], so no third word is touched. Steps whose four positions are all admissible run
// without masking; the last, partial step masks once. The case flag is a template parameter (no per-word flag tests).
template <uint32_t HFLAGS>
TPLX_HD int64_t str_find_impl(const StrV &h, const StrV &n) {
    const uint32_t last = h.len - n.len;  // last admissible start
    const uint32_t c0 = sch(n, 0) * 0x01010101u;
    const bool two = n.len >= 2;
    const uint32_t c1 = (two ? sch(n, 1) : 0) * 0x01010101u;
    const uintptr_t addr = (uintptr_t)h.p;
    const uint32_t *aw = (const uint32_t *)(addr & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(addr & 3) * 8;
    const uint32_t nwords = (uint32_t)(((addr & 3) + h.len + 3) >> 2);  // aligned words holding string bytes (>= 1)
    const uint32_t kfull = (last + 1) >> 2;                             // steps k < kfull: positions 4k..4k+3 are all <= last
    const uint32_t rem = (last + 1) & 3;                                // admissible positions of the partial step kfull
    const uint32_t nsteps = kfull + (rem ? 1 : 0);
    const uint32_t tail_mask = (1u << (8 * rem)) - 1u;                  // rem in 1..3
    const bool plain_needle = n.flags == TPLX_SF_NONE;
    uint32_t a0 = aw[0];
    for (uint32_t k = 0; k < nsteps; ++k) {
        // aw[k+1] holds string bytes whenever it is used: for sh != 0 it completes string word k; for a 2-character needle it holds
        // character 4k+4 <= last + 1 < h.len (full step). The bounds test only matters for the partial step / a 1-character needle.
        const uint32_t a1 = (k + 1 < nwords) ? aw[k + 1] : 0u;
        const uint32_t cur = case4_t<HFLAGS>(funnel_r(a0, a1, sh));
        uint32_t m;
        if (two) {
            const uint32_t nx = case4_t<HFLAGS>(a1 >> sh);  // low byte = character 4k+4
            m = both_zero4(cur ^ c0, ((cur >> 8) | (nx << 24)) ^ c1);
        } else {
            m = both_zero4(cur ^ c0, 0u);
        }
        if (k >= kfull) m &= tail_mask;
        while (m) {
#ifdef __CUDA_ARCH__
            const uint32_t bit = __ffs(m) - 1;
#else
            const uint32_t bit = (uint32_t)__builtin_ctz(m);
#endif
            const uint32_t pos = 4 * k + (bit >> 3);
            bool ok = true;
            if (plain_needle) for (uint32_t j = two ? 2 : 1; ok && j < n.len; ++j) ok = sch_t<HFLAGS>(h.p, pos + j) == n.p[j];
            else for (uint32_t j = two ? 2 : 1; ok && j < n.len; ++j) ok = sch_t<HFLAGS>(h.p, pos + j) == sch(n, j);
            if (ok) return (int64_t)pos;
            m &= m - 1;
        }
        a0 = a1;
    }
    return -1;
}

TPLX_HD_NOINLINE int64_t str_find(StrV h, StrV n) {
    if (n.len == 0) return 0;
    if (n.len > h.len) return -1;
    if (h.flags == TPLX_SF_LOWER) return str_find_impl<TPLX_SF_LOWER>(h, n);
    if (h.flags == TPLX_SF_UPPER) return str_find_impl<TPLX_SF_UPPER>(h, n);
    return str_find_impl<TPLX_SF_NONE>(h, n);
}

// std::string::rfind: last occurrence or -1; empty needle -> len.
// Same SWAR filter as str_find, walking the haystack backwards four positions per step (one new aligned load per step).
template <uint32_t HFLAGS>
TPLX_HD int64_t str_rfind_impl(const StrV &h, const StrV &n) {
    const uint32_t last = h.len - n.len;  // last admissible start
    const uint32_t c0 = sch(n, 0);
    const bool two = n.len >= 2;
    const uint32_t c1 = two ? sch(n, 1) : 0;
    const uintptr_t addr = (uintptr_t)h.p;
    const uint32_t *aw = (const uint32_t *)(addr & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(addr & 3) * 8;
    const uint32_t nwords = (uint32_t)(((addr & 3) + h.len + 3) >> 2);  // aligned words holding string bytes (>= 1)
    int32_t k = (int32_t)(last >> 2);                                    // string word (characters 4k..4k+3) that holds position `last`
    uint32_t hi1 = ((uint32_t)k + 1 < nwords) ? aw[k + 1] : 0u;
    const uint32_t hi2 = ((uint32_t)k + 2 < nwords) ? aw[k + 2] : 0u;
    uint32_t nxt = funnel_r(hi1, hi2, sh);  // string word k+1: only its first character is needed (2-character test of position 4k+3)
    if (HFLAGS == TPLX_SF_LOWER) nxt = lower4(nxt);
    if (HFLAGS == TPLX_SF_UPPER) nxt = upper4(nxt);
    for (; k >= 0; --k) {
        const uint32_t lo = aw[k];
        uint32_t cur = funnel_r(lo, hi1, sh);
        if (HFLAGS == TPLX_SF_LOWER) cur = lower4(cur);
        if (HFLAGS == TPLX_SF_UPPER) cur = upper4(cur);
        uint32_t m = eq_mask4(cur, c0);
        if (two) m &= eq_mask4((cur >> 8) | (nxt << 24), c1);
        const uint32_t valid = last - 4 * (uint32_t)k;  // positions 0..valid of this word are admissible
        if (valid < 3) m &= low_mask(valid + 1);
        while (m) {
#ifdef __CUDA_ARCH__
            const uint32_t bit = 31u - (uint32_t)__clz((int)m);
#else
            const uint32_t bit = 31u - (uint32_t)__builtin_clz(m);
#endif
            const uint32_t pos = 4 * (uint32_t)k + (bit >> 3);
            if (match_at(h, pos, n, two ? 2 : 1)) return (int64_t)pos;
            m ^= 1u << bit;
        }
        nxt = cur;
        hi1 = lo;
    }
    return -1;
}

TPLX_HD_NOINLINE int64_t str_rfind(StrV h, StrV n) {
    if (n.len > h.len) return -1;
    if (n.len == 0) return (int64_t)h.len;
    if (h.flags == TPLX_SF_LOWER) return str_rfind_impl<TPLX_SF_LOWER>(h, n);
    if (h.flags == TPLX_SF_UPPER) return str_rfind_impl<TPLX_SF_UPPER>(h, n);
    return str_rfind_impl<TPLX_SF_NONE>(h, n);
}

TPLX_HD bool is_pyspace(uint8_t c) {
    // string.whitespace = ' \t\n\r\x0b\x0c' (runtime/src/Runtime.cc:322-333)
    return c == ' ' || (c >= 9 && c <= 13);
}

// Python slice index normalisation for stride +1 (BlockGeneratorVisitor.cc:4618-4690)
TPLX_HD int64_t slice_index(int64_t idx, int64_t len) {
    if (idx < -len) return 0;
    if (idx <= -1) return idx + len;
    if (idx < len) return idx;
    return len;
}

// fast_atoi64 (runtime/src/Runtime.cc:319-341 + utils/src/StringUtils.cc:22-63); false = ValueError
TPLX_HD bool str_to_i64(const StrV &s, int64_t *out) {
    uint32_t i = 0, e = s.len;
    while (i < e && is_pyspace(s.p[i])) ++i;
    if (e > i) {
        uint32_t e2 = e - 1;
        while (e2 > i && is_pyspace(s.p[e2])) --e2;
        e = e2 + 1;
    }
    if (i == e) return false;
    bool neg = false;
    if (s.p[i] == '-') {
        neg = true;
        ++i;
    }
    uint64_t x = 0;
    while (i < s.len) {
        uint8_t d = (uint8_t)(s.p[i] - '0');
        if (d > 9) break;
        x = x * 10 + d;
        ++i;
    }
    if (i != e) return false;
    *out = (int64_t)(neg ? (uint64_t)0 - x : x);
    return true;
}

// floor division / modulo with sign fix-up (codegen/src/LLVMEnvironment.cc:1377-1430)
TPLX_HD int64_t floordiv_i64(int64_t x, int64_t y) {
    int64_t q = x / y, r = x % y;
    if (r != 0 && ((r < 0) != (y < 0))) --q;
    return q;
}
TPLX_HD int64_t floormod_i64(int64_t x, int64_t y) {
    int64_t r = x % y;
    if (r != 0 && ((r < 0) != (y < 0))) r += y;
    return r;
}

}  // namespace tplx
