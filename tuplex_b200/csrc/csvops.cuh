// csvops.cuh — CSV row machine and cell decoders (K6), host + device.
//
// Restated from the reference's default CSV source (paths relative to /root/reference/tuplex/):
//   row / cell splitting   csvmonkey::CsvReader::try_parse      core/include/physical/csvmonkey.h:523-672
//   cell dequoting         csvmonkey::CsvCell::as_str            core/include/physical/csvmonkey.h:320-335
//   newline at EOF         VFCSVStreamCursor (appends '\n')      core/src/physical/CSVReader.cc:66-100,167-177
//   cells -> typed row     decodeCells                           codegen/src/FlattenedTuple.cc:1215-1330
//   int / float / bool     fast_atoi64, fast_atod, fast_atob     runtime/src/Runtime.cc:319-385, utils/src/StringUtils.cc:22-260
// The generated parser (core/src/physical/CSVParseRowGenerator.cc:436-760) splits rows the same way on the inputs its
// tests hold (test/core/CSVRowParseGeneratorTests.cc); those tests are this file's known-answer vectors.
//
// Buffer contract: positions are uint32; the caller guarantees buf[n] == '\n' (the newline the reference's cursor
// appends), so every scan below terminates at or before position n.
//
// Compiles for the host as well (tests/test_csv_host.py fuzzes these exact functions against the oracle).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "strops.cuh"

namespace tplx {

constexpr uint32_t CSV_UNDERRUN = 0xFFFFFFFFu;  // input ended inside a quoted cell: csvmonkey yields no row
constexpr uint32_t CSV_DEQ_CAP = 64;            // local buffer for escaped numeric cells

#ifdef __CUDA_ARCH__
#define TPLX_DMUL(a, b) __dmul_rn((a), (b))
#define TPLX_DADD(a, b) __dadd_rn((a), (b))
#define TPLX_DDIV(a, b) __ddiv_rn((a), (b))
#else  // host build uses -ffp-contract=off
#define TPLX_DMUL(a, b) ((a) * (b))
#define TPLX_DADD(a, b) ((a) + (b))
#define TPLX_DDIV(a, b) ((a) / (b))
#endif

TPLX_HD bool csv_is_nl(uint8_t c) { return c == '\n' || c == '\r'; }

// ---- 8 bytes at a time (little endian). Buffers are padded past [n], so the aligned word holding any position <= n
// may be read whole.
TPLX_HD uint64_t csv_load8(const uint8_t *p) {  // p is 8-byte aligned on the device
#ifdef __CUDA_ARCH__
    return *reinterpret_cast<const uint64_t *>(p);
#else
    uint64_t w = 0;
    for (int k = 7; k >= 0; --k) w = (w << 8) | p[k];
    return w;
#endif
}
// 0x80 in every byte lane of w that equals c (exact)
TPLX_HD uint64_t csv_eq8(uint64_t w, uint8_t c) {
    const uint64_t x = w ^ (0x0101010101010101ull * c);
    const uint64_t t = ((x & 0x7f7f7f7f7f7f7f7full) + 0x7f7f7f7f7f7f7f7full) | x;
    return ~t & 0x8080808080808080ull;
}
// lane mask (0x80 per byte) -> 8 bits, bit i = byte i
TPLX_HD uint32_t csv_pack8(uint64_t m) { return (uint32_t)(((m >> 7) * 0x0102040810204080ull) >> 56); }
TPLX_HD uint32_t csv_ctz64(uint64_t m) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__ffsll((long long)m) - 1;
#else
    return (uint32_t)__builtin_ctzll(m);
#endif
}
// first position >= p whose byte is a, b or c; the caller guarantees one exists at or before [n] (the appended newline)
TPLX_HD uint32_t csv_find3(const uint8_t *buf, uint32_t p, uint8_t a, uint8_t b, uint8_t c) {
    uint32_t base = p & ~7u;
    uint64_t w = csv_load8(buf + base);
    uint64_t m = (csv_eq8(w, a) | csv_eq8(w, b) | csv_eq8(w, c)) & (~0ull << (8 * (p & 7)));
    while (!m) {
        base += 8;
        w = csv_load8(buf + base);
        m = csv_eq8(w, a) | csv_eq8(w, b) | csv_eq8(w, c);
    }
    return base + (csv_ctz64(m) >> 3);
}
// first position in [p, n] whose byte is q, or a value > n
TPLX_HD uint32_t csv_find1(const uint8_t *buf, uint32_t p, uint32_t n, uint8_t q) {
    uint32_t base = p & ~7u;
    uint64_t m = csv_eq8(csv_load8(buf + base), q) & (~0ull << (8 * (p & 7)));
    while (!m) {
        base += 8;
        if (base > n) return n + 1;
        m = csv_eq8(csv_load8(buf + base), q);
    }
    return base + (csv_ctz64(m) >> 3);
}

// Runs the row machine from p (first byte of the row, never a newline). f(cell_index, begin, end, escaped) is
// called for every cell ([begin,end) = raw content, quotes of a quoted cell excluded). Returns the position of
// the row's terminating newline and the number of cells, or CSV_UNDERRUN.
template <class F>
TPLX_HD uint32_t csv_row_machine(const uint8_t *buf, uint32_t p, uint32_t n, uint8_t delim, uint8_t quote, uint32_t *ncells,
                                 F &&f) {
    uint32_t cell = 0;
    for (;;) {
        uint8_t c = buf[p];
        if (csv_is_nl(c)) {  // newline right after a delimiter: empty final cell (csvmonkey.h:567-577)
            f(cell, p, p, false);
            *ncells = cell + 1;
            return p;
        }
        if (c == quote) {
            const uint32_t b = ++p;
            bool esc = false;
            for (;;) {
                p = csv_find1(buf, p, n, quote);
                if (p >= n) return CSV_UNDERRUN;  // buf[n] is the appended newline, never a quote
                const uint32_t q = p++;           // p = byte after the quote (<= n)
                c = buf[p];
                if (c == delim) {
                    f(cell, b, q, esc);
                    ++cell;
                    ++p;
                    break;
                }
                if (csv_is_nl(c)) {
                    f(cell, b, q, esc);
                    *ncells = cell + 1;
                    return p;
                }
                esc = true;  // doubled quote or stray quote: the following byte is skipped (csvmonkey.h:619-623)
                ++p;
            }
        } else {
            const uint32_t b = p;
            p = csv_find3(buf, p, delim, '\n', '\r');
            f(cell, b, p, false);
            if (buf[p] == delim) {
                ++cell;
                ++p;
            } else {
                *ncells = cell + 1;
                return p;
            }
        }
    }
}

// as_str(): every quote character is dropped and the byte after it copied verbatim
TPLX_HD uint32_t csv_dequoted_len(const uint8_t *buf, uint32_t b, uint32_t e, uint8_t quote) {
    uint32_t o = 0;
    for (uint32_t i = b; i < e; ++i) {
        if (buf[i] == quote) {
            ++i;
            if (i >= e) break;
        }
        ++o;
    }
    return o;
}
TPLX_HD uint32_t csv_dequote(const uint8_t *buf, uint32_t b, uint32_t e, uint8_t quote, uint8_t *out, uint32_t cap) {
    uint32_t o = 0;
    for (uint32_t i = b; i < e; ++i) {
        if (buf[i] == quote) {
            ++i;
            if (i >= e) break;
        }
        if (o < cap) out[o] = buf[i];
        ++o;
    }
    return o;
}

// dequoted cell == s ?
TPLX_HD bool csv_cell_equals(const uint8_t *buf, uint32_t b, uint32_t e, bool escaped, uint8_t quote, const uint8_t *s,
                             uint32_t slen) {
    if (!escaped) {
        if (e - b != slen) return false;
        for (uint32_t i = 0; i < slen; ++i)
            if (buf[b + i] != s[i]) return false;
        return true;
    }
    uint32_t o = 0;
    for (uint32_t i = b; i < e; ++i) {
        if (buf[i] == quote) {
            ++i;
            if (i >= e) break;
        }
        if (o >= slen || buf[i] != s[o]) return false;
        ++o;
    }
    return o == slen;
}

// whitespace trimming shared by the runtime wrappers (Runtime.cc:319-341,343-365): [i, e) of p[0..len)
// The decoders read the cell through an accessor get(k) -> byte k, so that the same code runs over memory (host tests,
// escaped cells) and over a cell held in registers (CsvCell32 below).
template <class G>
TPLX_HD void csv_trim_g(G &&get, uint32_t len, uint32_t *pi, uint32_t *pe) {
    uint32_t i = 0, e = len;
    while (i < e && is_pyspace(get(i))) ++i;
    if (e > i) {
        uint32_t e2 = e - 1;
        while (e2 > i && is_pyspace(get(e2))) --e2;
        e = e2 + 1;
    }
    *pi = i;
    *pe = e;
}

// A cell of at most 32 bytes in four registers: five independent aligned loads instead of one dependent byte load per
// character (csv_parse_rows is latency-bound on those).
struct CsvCell32 {
    uint64_t w0, w1, w2, w3;
    TPLX_HD void load(const uint8_t *buf, uint32_t b) {
        const uint32_t base = b & ~7u, sh = (b & 7u) * 8;
        const uint64_t a0 = csv_load8(buf + base), a1 = csv_load8(buf + base + 8), a2 = csv_load8(buf + base + 16),
                       a3 = csv_load8(buf + base + 24), a4 = csv_load8(buf + base + 32);
        if (sh) {
            w0 = (a0 >> sh) | (a1 << (64 - sh));
            w1 = (a1 >> sh) | (a2 << (64 - sh));
            w2 = (a2 >> sh) | (a3 << (64 - sh));
            w3 = (a3 >> sh) | (a4 << (64 - sh));
        } else {
            w0 = a0, w1 = a1, w2 = a2, w3 = a3;
        }
    }
    TPLX_HD uint8_t get(uint32_t k) const {  // k < 32
        const uint64_t w = k < 16 ? (k < 8 ? w0 : w1) : (k < 24 ? w2 : w3);
        return (uint8_t)(w >> (8 * (k & 7)));
    }
};

// (double)d / 10^k for d = 0..9, k = 1..22, computed exactly as fast_atod does at run time (pow10 = 10.0; pow10 *= 10.0 per
// digit — exact up to 10^22 — and one IEEE division): the quotients are fixed doubles, so the device reads them instead of
// dividing (an f64 division costs tens of instructions). Generated by a 6-line Python loop (float.hex of d / pow10).
#define CSV_FRAC_KMAX 22
#ifdef __CUDA_ARCH__
__device__
#endif
static const double csv_frac_tab[CSV_FRAC_KMAX * 10] = {
    0x0p+0, 0x1.999999999999ap-4, 0x1.999999999999ap-3, 0x1.3333333333333p-2, 0x1.999999999999ap-2, 0x1.0000000000000p-1, 0x1.3333333333333p-1, 0x1.6666666666666p-1, 0x1.999999999999ap-1, 0x1.ccccccccccccdp-1,
    0x0p+0, 0x1.47ae147ae147bp-7, 0x1.47ae147ae147bp-6, 0x1.eb851eb851eb8p-6, 0x1.47ae147ae147bp-5, 0x1.999999999999ap-5, 0x1.eb851eb851eb8p-5, 0x1.1eb851eb851ecp-4, 0x1.47ae147ae147bp-4, 0x1.70a3d70a3d70ap-4,
    0x0p+0, 0x1.0624dd2f1a9fcp-10, 0x1.0624dd2f1a9fcp-9, 0x1.89374bc6a7efap-9, 0x1.0624dd2f1a9fcp-8, 0x1.47ae147ae147bp-8, 0x1.89374bc6a7efap-8, 0x1.cac083126e979p-8, 0x1.0624dd2f1a9fcp-7, 0x1.26e978d4fdf3bp-7,
    0x0p+0, 0x1.a36e2eb1c432dp-14, 0x1.a36e2eb1c432dp-13, 0x1.3a92a30553261p-12, 0x1.a36e2eb1c432dp-12, 0x1.0624dd2f1a9fcp-11, 0x1.3a92a30553261p-11, 0x1.6f0068db8bac7p-11, 0x1.a36e2eb1c432dp-11, 0x1.d7dbf487fcb92p-11,
    0x0p+0, 0x1.4f8b588e368f1p-17, 0x1.4f8b588e368f1p-16, 0x1.f75104d551d69p-16, 0x1.4f8b588e368f1p-15, 0x1.a36e2eb1c432dp-15, 0x1.f75104d551d69p-15, 0x1.2599ed7c6fbd2p-14, 0x1.4f8b588e368f1p-14, 0x1.797cc39ffd60fp-14,
    0x0p+0, 0x1.0c6f7a0b5ed8dp-20, 0x1.0c6f7a0b5ed8dp-19, 0x1.92a737110e454p-19, 0x1.0c6f7a0b5ed8dp-18, 0x1.4f8b588e368f1p-18, 0x1.92a737110e454p-18, 0x1.d5c31593e5fb7p-18, 0x1.0c6f7a0b5ed8dp-17, 0x1.2dfd694ccab3fp-17,
    0x0p+0, 0x1.ad7f29abcaf48p-24, 0x1.ad7f29abcaf48p-23, 0x1.421f5f40d8376p-22, 0x1.ad7f29abcaf48p-22, 0x1.0c6f7a0b5ed8dp-21, 0x1.421f5f40d8376p-21, 0x1.77cf44765195fp-21, 0x1.ad7f29abcaf48p-21, 0x1.e32f0ee144531p-21,
    0x0p+0, 0x1.5798ee2308c3ap-27, 0x1.5798ee2308c3ap-26, 0x1.01b2b29a4692bp-25, 0x1.5798ee2308c3ap-25, 0x1.ad7f29abcaf48p-25, 0x1.01b2b29a4692bp-24, 0x1.2ca5d05ea7ab3p-24, 0x1.5798ee2308c3ap-24, 0x1.828c0be769dc1p-24,
    0x0p+0, 0x1.12e0be826d695p-30, 0x1.12e0be826d695p-29, 0x1.9c511dc3a41dfp-29, 0x1.12e0be826d695p-28, 0x1.5798ee2308c3ap-28, 0x1.9c511dc3a41dfp-28, 0x1.e1094d643f784p-28, 0x1.12e0be826d695p-27, 0x1.353cd652bb167p-27,
    0x0p+0, 0x1.b7cdfd9d7bdbbp-34, 0x1.b7cdfd9d7bdbbp-33, 0x1.49da7e361ce4cp-32, 0x1.b7cdfd9d7bdbbp-32, 0x1.12e0be826d695p-31, 0x1.49da7e361ce4cp-31, 0x1.80d43de9cc603p-31, 0x1.b7cdfd9d7bdbbp-31, 0x1.eec7bd512b572p-31,
    0x0p+0, 0x1.5fd7fe1796495p-37, 0x1.5fd7fe1796495p-36, 0x1.07e1fe91b0b70p-35, 0x1.5fd7fe1796495p-35, 0x1.b7cdfd9d7bdbbp-35, 0x1.07e1fe91b0b70p-34, 0x1.33dcfe54a3803p-34, 0x1.5fd7fe1796495p-34, 0x1.8bd2fdda89128p-34,
    0x0p+0, 0x1.19799812dea11p-40, 0x1.19799812dea11p-39, 0x1.a636641c4df1ap-39, 0x1.19799812dea11p-38, 0x1.5fd7fe1796495p-38, 0x1.a636641c4df1ap-38, 0x1.ec94ca210599ep-38, 0x1.19799812dea11p-37, 0x1.3ca8cb153a753p-37,
    0x0p+0, 0x1.c25c268497682p-44, 0x1.c25c268497682p-43, 0x1.51c51ce3718e1p-42, 0x1.c25c268497682p-42, 0x1.19799812dea11p-41, 0x1.51c51ce3718e1p-41, 0x1.8a10a1b4047b2p-41, 0x1.c25c268497682p-41, 0x1.faa7ab552a552p-41,
    0x0p+0, 0x1.6849b86a12b9bp-47, 0x1.6849b86a12b9bp-46, 0x1.0e374a4f8e0b4p-45, 0x1.6849b86a12b9bp-45, 0x1.c25c268497682p-45, 0x1.0e374a4f8e0b4p-44, 0x1.3b40815cd0628p-44, 0x1.6849b86a12b9bp-44, 0x1.9552ef775510ep-44,
    0x0p+0, 0x1.203af9ee75616p-50, 0x1.203af9ee75616p-49, 0x1.b05876e5b0120p-49, 0x1.203af9ee75616p-48, 0x1.6849b86a12b9bp-48, 0x1.b05876e5b0120p-48, 0x1.f86735614d6a6p-48, 0x1.203af9ee75616p-47, 0x1.4442592c440d8p-47,
    0x0p+0, 0x1.cd2b297d889bcp-54, 0x1.cd2b297d889bcp-53, 0x1.59e05f1e2674dp-52, 0x1.cd2b297d889bcp-52, 0x1.203af9ee75616p-51, 0x1.59e05f1e2674dp-51, 0x1.9385c44dd7885p-51, 0x1.cd2b297d889bcp-51, 0x1.036847569cd7ap-50,
    0x0p+0, 0x1.70ef54646d497p-57, 0x1.70ef54646d497p-56, 0x1.14b37f4b51f71p-55, 0x1.70ef54646d497p-55, 0x1.cd2b297d889bcp-55, 0x1.14b37f4b51f71p-54, 0x1.42d169d7dfa04p-54, 0x1.70ef54646d497p-54, 0x1.9f0d3ef0faf29p-54,
    0x0p+0, 0x1.2725dd1d243acp-60, 0x1.2725dd1d243acp-59, 0x1.bab8cbabb6581p-59, 0x1.2725dd1d243acp-58, 0x1.70ef54646d497p-58, 0x1.bab8cbabb6581p-58, 0x1.024121797fb36p-57, 0x1.2725dd1d243acp-57, 0x1.4c0a98c0c8c21p-57,
    0x0p+0, 0x1.d83c94fb6d2acp-64, 0x1.d83c94fb6d2acp-63, 0x1.622d6fbc91e01p-62, 0x1.d83c94fb6d2acp-62, 0x1.2725dd1d243acp-61, 0x1.622d6fbc91e01p-61, 0x1.9d35025bff857p-61, 0x1.d83c94fb6d2acp-61, 0x1.09a213cd6d681p-60,
    0x0p+0, 0x1.79ca10c924223p-67, 0x1.79ca10c924223p-66, 0x1.1b578c96db19bp-65, 0x1.79ca10c924223p-65, 0x1.d83c94fb6d2acp-65, 0x1.1b578c96db19bp-64, 0x1.4a90ceafff9dfp-64, 0x1.79ca10c924223p-64, 0x1.a90352e248a68p-64,
    0x0p+0, 0x1.2e3b40a0e9b4fp-70, 0x1.2e3b40a0e9b4fp-69, 0x1.c558e0f15e8f7p-69, 0x1.2e3b40a0e9b4fp-68, 0x1.79ca10c924223p-68, 0x1.c558e0f15e8f7p-68, 0x1.0873d88ccc7e6p-67, 0x1.2e3b40a0e9b4fp-67, 0x1.5402a8b506eb9p-67,
    0x0p+0, 0x1.e392010175ee6p-74, 0x1.e392010175ee6p-73, 0x1.6aad80c11872cp-72, 0x1.e392010175ee6p-72, 0x1.2e3b40a0e9b4fp-71, 0x1.6aad80c11872cp-71, 0x1.a71fc0e147309p-71, 0x1.e392010175ee6p-71, 0x1.10022090d2561p-70};

// fast_atod (StringUtils.cc:71-163) behind the runtime wrapper's trim; false = ValueError.
// The accumulation is the reference's own (not correctly rounded): value = 10*value + d; value += d / pow10.
template <class G>
TPLX_HD bool csv_atod_g(G &&get, uint32_t len, double *out) {
    uint32_t i0, e;
    csv_trim_g(get, len, &i0, &e);
    if (i0 == e) return false;
    // bytes at or past e never match a digit, sign, '.', 'e' or a letter of nan/infinity in the reference either
    // (there it is whitespace or the terminator), so they read as 0 here
#define CH(k) ((k) < e ? get(k) : (uint8_t)0)
    uint32_t p = i0;
    double sign = 1.0;
    if (CH(p) == '-') {
        sign = -1.0;
        ++p;
    } else if (CH(p) == '+')
        ++p;
    double value = 0.0;
    for (; (uint8_t)(CH(p) - '0') <= 9; ++p) value = TPLX_DADD(TPLX_DMUL(10.0, value), (double)(CH(p) - '0'));
    if (CH(p) == '.') {
        double pow10 = 10.0;
        uint32_t k = 0;  // fraction digits seen
        ++p;
        while ((uint8_t)(CH(p) - '0') <= 9) {
            const uint32_t d = (uint32_t)(CH(p) - '0');
            if (k < CSV_FRAC_KMAX)
                value = TPLX_DADD(value, csv_frac_tab[k * 10 + d]);
            else
                value = TPLX_DADD(value, TPLX_DDIV((double)d, pow10));
            pow10 = TPLX_DMUL(pow10, 10.0);
            ++k;
            ++p;
        }
    }
    int frac = 0;
    double scale = 1.0;
    if (CH(p) == 'e' || CH(p) == 'E') {
        uint32_t exponent = 0;
        ++p;
        if (CH(p) == '-') {
            frac = 1;
            ++p;
        } else if (CH(p) == '+')
            ++p;
        for (; (uint8_t)(CH(p) - '0') <= 9; ++p) exponent = exponent * 10u + (uint32_t)(CH(p) - '0');
        if (exponent > 308) exponent = 308;
        while (exponent >= 50) {
            scale = TPLX_DMUL(scale, 1E50);
            exponent -= 50;
        }
        while (exponent >= 8) {
            scale = TPLX_DMUL(scale, 1E8);
            exponent -= 8;
        }
        while (exponent > 0) {
            scale = TPLX_DMUL(scale, 10.0);
            exponent -= 1;
        }
    }
    int nanmatch = 0, infmatch = 0;
    if (p == i0) {
        const char *nanstr = "nan";
        while (nanmatch < 3 && (CH(p) == (uint8_t)nanstr[nanmatch] || CH(p) == (uint8_t)(nanstr[nanmatch] - 32))) {
            ++p;
            ++nanmatch;
        }
    }
    if (p == i0) {
        const char *infstr = "infinity";
        while (infmatch < 8 && (CH(p) == (uint8_t)infstr[infmatch] || CH(p) == (uint8_t)(infstr[infmatch] - 32))) {
            ++p;
            ++infmatch;
        }
    }
#undef CH
    if (p != e) return false;
    if (nanmatch == 3) {
        uint64_t bits = 0x7FF8000000000000ull;  // NAN
        *out = *reinterpret_cast<double *>(&bits);
    } else if (infmatch == 3 || infmatch == 8) {
        uint64_t bits = 0x7FF0000000000000ull;  // +INFINITY (the sign is not applied, StringUtils.cc:155)
        *out = *reinterpret_cast<double *>(&bits);
    } else {
        *out = TPLX_DMUL(sign, frac ? TPLX_DDIV(value, scale) : TPLX_DMUL(value, scale));
    }
    return true;
}

TPLX_HD bool csv_atod(const uint8_t *s, uint32_t len, double *out) {
    return csv_atod_g([s](uint32_t k) { return s[k]; }, len, out);
}

// fast_atoi64 (StringUtils.cc:22-63) behind the runtime wrapper's trim (Runtime.cc:319-341); accessor twin of str_to_i64
template <class G>
TPLX_HD bool csv_atoi64_g(G &&get, uint32_t len, int64_t *out) {
    uint32_t i, e;
    csv_trim_g(get, len, &i, &e);
    if (i == e) return false;
    bool neg = false;
    if (get(i) == '-') {
        neg = true;
        ++i;
    }
    uint64_t x = 0;
    while (i < len) {  // like str_to_i64: digits may run up to the end of the cell, then the position must equal e
        const uint8_t d = (uint8_t)(get(i) - '0');
        if (d > 9) break;
        x = x * 10 + d;
        ++i;
    }
    if (i != e) return false;
    *out = (int64_t)(neg ? (uint64_t)0 - x : x);
    return true;
}

// fast_atob (StringUtils.cc:180-255): no trimming; t/y/f/n, no, yes, true, false — case-insensitive
template <class G>
TPLX_HD bool csv_atob_g(G &&get, uint32_t len, int64_t *out) {
    uint8_t b[5];
    if (len == 0 || len > 5) return false;
    for (uint32_t i = 0; i < len; ++i) b[i] = case1(get(i), TPLX_SF_LOWER);
    switch (len) {
        case 1:
            if (b[0] == 'y' || b[0] == 't') {
                *out = 1;
                return true;
            }
            if (b[0] == 'n' || b[0] == 'f') {
                *out = 0;
                return true;
            }
            return false;
        case 2:
            if (b[0] == 'n' && b[1] == 'o') {
                *out = 0;
                return true;
            }
            return false;
        case 3:
            if (b[0] == 'y' && b[1] == 'e' && b[2] == 's') {
                *out = 1;
                return true;
            }
            return false;
        case 4:
            if (b[0] == 't' && b[1] == 'r' && b[2] == 'u' && b[3] == 'e') {
                *out = 1;
                return true;
            }
            return false;
        default:
            if (b[0] == 'f' && b[1] == 'a' && b[2] == 'l' && b[3] == 's' && b[4] == 'e') {
                *out = 0;
                return true;
            }
            return false;
    }
}

TPLX_HD bool csv_atob(const uint8_t *s, uint32_t len, int64_t *out) {
    return csv_atob_g([s](uint32_t k) { return s[k]; }, len, out);
}

// what a selected column needs from one cell
struct CsvNulls {
    uint8_t n;
    uint8_t off[9];     // value k = bytes[off[k], off[k+1])
    uint8_t bytes[64];
};

TPLX_HD bool csv_cell_is_null(const uint8_t *buf, uint32_t b, uint32_t e, bool escaped, uint8_t quote, const CsvNulls &nv) {
    for (uint32_t k = 0; k < nv.n; ++k)
        if (csv_cell_equals(buf, b, e, escaped, quote, nv.bytes + nv.off[k], (uint32_t)(nv.off[k + 1] - nv.off[k]))) return true;
    return false;
}

// typed decode of one numeric / bool cell -> 64-bit slot value; false = conversion error
TPLX_HD bool csv_decode_scalar(const uint8_t *buf, uint32_t b, uint32_t e, bool escaped, uint8_t quote, uint8_t type,
                               uint64_t *bits) {
    uint8_t tmp[CSV_DEQ_CAP];
    const uint8_t *p = buf + b;
    uint32_t len = e - b;
    if (escaped) {
        len = csv_dequote(buf, b, e, quote, tmp, CSV_DEQ_CAP);
        if (len > CSV_DEQ_CAP) return false;  // left to the interpreter path
        p = tmp;
    }
    if (!escaped && len <= 32) {  // the common case: decode from registers
        CsvCell32 cell;
        cell.load(buf, b);
        auto get = [&cell](uint32_t k) { return cell.get(k); };
        if (type == TPLX_T_I64) {
            int64_t v;
            if (!csv_atoi64_g(get, len, &v)) return false;
            *bits = (uint64_t)v;
            return true;
        }
        if (type == TPLX_T_F64) {
            double d;
            if (!csv_atod_g(get, len, &d)) return false;
            *bits = *reinterpret_cast<uint64_t *>(&d);
            return true;
        }
        int64_t bv;
        if (!csv_atob_g(get, len, &bv)) return false;
        *bits = (uint64_t)bv;
        return true;
    }
    auto getm = [p](uint32_t k) { return p[k]; };
    if (type == TPLX_T_I64) {
        int64_t v;
        if (!csv_atoi64_g(getm, len, &v)) return false;
        *bits = (uint64_t)v;
        return true;
    }
    if (type == TPLX_T_F64) {
        double d;
        if (!csv_atod_g(getm, len, &d)) return false;
        *bits = *reinterpret_cast<uint64_t *>(&d);
        return true;
    }
    int64_t bv;
    if (!csv_atob_g(getm, len, &bv)) return false;
    *bits = (uint64_t)bv;
    return true;
}

// ---- row finding by quote parity ------------------------------------------------------------------
constexpr uint32_t CSV_SPAN = 64;  // bytes walked by one thread
constexpr uint32_t CSV_SKIP = 0xFF;

struct CsvState {
    uint32_t par;  // quotes in the span, mod 2
    uint32_t c0;   // row ends in the span if it starts outside quotes
    uint32_t c1;   // ... if it starts inside quotes
};
TPLX_HD CsvState csv_compose(const CsvState &a, const CsvState &b) {
    CsvState r;
    r.par = a.par ^ b.par;
    r.c0 = a.c0 + (a.par ? b.c1 : b.c0);
    r.c1 = a.c1 + (a.par ? b.c0 : b.c1);
    return r;
}

// A newline ends a row iff it lies outside quotes and the byte before it is not a newline (blank lines and the '\n'
// of "\r\n" are skipped at row start, csvmonkey.h:551-561). The buffer is zero padded to a span multiple, so spans
// need no bounds checks (NUL is neither quote nor newline). emit(pos) is called for every row end when the span's
// start parity is par0 (pass a value > 1 to only count).
template <class Emit>
TPLX_HD CsvState csv_walk_span(const uint8_t *buf, uint64_t start, uint8_t quote, uint32_t par0, Emit &&emit) {
    CsvState s{0, 0, 0};
    uint32_t par = 0;                                                              // quotes so far in the span, mod 2
    uint32_t prev_nl = start == 0 ? 1u : (csv_is_nl(buf[start - 1]) ? 1u : 0u);  // is the previous byte a newline
    const uint32_t flip0 = par0 == 1 ? 0xFFu : 0u;
    for (uint32_t k = 0; k < CSV_SPAN / 8; ++k) {
        const uint64_t w = csv_load8(buf + start + 8 * k);
        const uint32_t q = csv_pack8(csv_eq8(w, quote));
        const uint32_t nl = csv_pack8(csv_eq8(w, '\n') | csv_eq8(w, '\r'));
        uint32_t x = q;  // inclusive prefix parity of the quote bits
        x ^= x << 1;
        x ^= x << 2;
        x ^= x << 4;
        const uint32_t inside = (x ^ (par ? 0xFFu : 0u)) & 0xFFu;  // relative to a span that starts outside quotes
        const uint32_t cand = nl & ~((nl << 1) | prev_nl) & 0xFFu;  // newline whose previous byte is not one
#ifdef __CUDA_ARCH__
        s.c1 += __popc(cand & inside);
        s.c0 += __popc(cand & ~inside);
#else
        s.c1 += (uint32_t)__builtin_popcount(cand & inside);
        s.c0 += (uint32_t)__builtin_popcount(cand & ~inside & 0xFFu);
#endif
        if (par0 <= 1) {
            uint32_t e = cand & ~(inside ^ flip0) & 0xFFu;  // outside quotes given the real start parity
            while (e) {
                const uint32_t i = csv_ctz64(e);
                emit(start + 8 * k + i);
                e &= e - 1;
            }
        }
        par = (inside >> 7) & 1u;
        prev_nl = (nl >> 7) & 1u;
    }
    s.par = par;
    return s;
}

// ---- one row: machine + decode + verification of the predicted row end --------------------------------
struct CsvParseParams {
    const uint8_t *buf;
    uint32_t n;  // data bytes; buf[n] == '\n'
    const uint32_t *row_end;
    uint32_t r0;  // first data row (1 when a header row is skipped)
    uint32_t nd;  // data rows
    uint8_t delim, quote;
    uint32_t n_file_cols;
    const uint8_t *col_kind;  // [n_file_cols] tplx_type or CSV_SKIP
    const uint8_t *col_slot;  // [n_file_cols] output column
    CsvNulls nulls;
    uint32_t n_out, n_str;
    uint8_t out_types[TPLX_MAX_COLS];
    int8_t strk[TPLX_MAX_COLS];
    uint64_t *tmp[TPLX_MAX_COLS];  // [nd] numeric: value bits; string: start | raw_len << 32 | escaped << 63
    uint64_t *lens;                // [n_str][nd + 1] dequoted lengths (scanned in place)
    uint64_t *good;                // [nd + 1] 1 = normal-case row (scanned in place)
    uint32_t *code;                // [nd] exception code, 0 = good
    uint32_t *flags;               // [0] != 0: a row did not end where quote parity predicted
    uint64_t *nullmask;            // [nd] bit k set = output column k (an Option column) is None in this row; null when no column is Option
};

TPLX_HD uint32_t csv_row_start(const uint8_t *buf, const uint32_t *row_end, uint32_t r) {
    uint32_t p = r == 0 ? 0u : row_end[r - 1] + 1;
    while (csv_is_nl(buf[p])) ++p;  // stops: row r has at least one non-newline byte before row_end[r]
    return p;
}

TPLX_HD void csv_parse_one_row(const CsvParseParams &P, uint32_t i) {
    const uint32_t r = P.r0 + i;
    const uint32_t start = csv_row_start(P.buf, P.row_end, r), end = P.row_end[r];
    uint32_t code = 0, ncells = 0;
    if (P.nullmask) P.nullmask[i] = 0;  // set bit by bit below: a mask held in a register across the row machine spills
    const uint32_t got = csv_row_machine(P.buf, start, P.n, P.delim, P.quote, &ncells, [&](uint32_t c, uint32_t b, uint32_t e, bool esc) {
        if (c >= P.n_file_cols || code) return;
        uint32_t kind = P.col_kind[c];
        if (kind == CSV_SKIP) return;
        const uint32_t slot = P.col_slot[c];
        if (csv_cell_is_null(P.buf, b, e, esc, P.quote, P.nulls)) {
            if (!(kind & TPLX_T_OPTION)) {
                code = TPLX_EC_NULLERROR;  // null in a non-Option column (FlattenedTuple.cc:1266-1279)
                return;
            }
            // None in an Option column (decodeCells, FlattenedTuple.cc:1259-1300): placeholder 0 / empty string, validity bit clear
            P.nullmask[i] |= 1ull << slot;
            P.tmp[slot][i] = 0;
            if (P.strk[slot] >= 0) P.lens[(size_t)P.strk[slot] * (P.nd + 1) + i] = 0;
            return;
        }
        kind &= ~TPLX_T_OPTION;
        if (kind == TPLX_T_STR) {
            P.tmp[slot][i] = (uint64_t)b | ((uint64_t)(e - b) << 32) | ((uint64_t)esc << 63);
            if (P.strk[slot] >= 0)  // lazy columns (strk < 0) keep the reference only
                P.lens[(size_t)P.strk[slot] * (P.nd + 1) + i] = esc ? csv_dequoted_len(P.buf, b, e, P.quote) : (e - b);
        } else {
            uint64_t bits = 0;
            if (!csv_decode_scalar(P.buf, b, e, esc, P.quote, (uint8_t)kind, &bits)) code = TPLX_EC_BADPARSE_STRING_INPUT;
            P.tmp[slot][i] = bits;
        }
    });
    if (got != end) {
        P.flags[0] = 1;  // speculation failed: the host switches to the sequential row finder
        code = TPLX_EC_BADPARSE_STRING_INPUT;
    }
    if (ncells != P.n_file_cols) code = TPLX_EC_BADPARSE_STRING_INPUT;  // checked before any cell is decoded (CSVReader.cc:470-479)
    if (code)
        for (uint32_t k = 0; k < P.n_str; ++k) P.lens[(size_t)k * (P.nd + 1) + i] = 0;
    P.code[i] = code;
    P.good[i] = code ? 0 : 1;
}

// exact, sequential row finding (repair path for irregular quoting); returns the number of rows
TPLX_HD uint32_t csv_find_rows_sequential(const uint8_t *buf, uint32_t n, uint8_t delim, uint8_t quote, uint32_t *row_end) {
    uint32_t p = 0, rows = 0;
    for (;;) {
        while (p <= n && csv_is_nl(buf[p])) ++p;
        if (p > n) break;
        uint32_t nc;
        const uint32_t e = csv_row_machine(buf, p, n, delim, quote, &nc, [](uint32_t, uint32_t, uint32_t, bool) {});
        if (e == CSV_UNDERRUN) break;
        row_end[rows++] = e;
        p = e + 1;
    }
    return rows;
}

// ---- CSV sink (K7): one output row as text --------------------------------------------------------------
// fast_csvwriter (core/src/physical/PipelineBuilder.cc:1550-1722): bool -> true / false, i64 -> decimal (i64toa),
// str -> quoteForCSV (runtime/src/Runtime.cc:682-738: quoted iff the cell holds a quote, the separator, '\n' or '\r';
// quotes doubled), a None cell of an Option column -> the null value quoted once (`null_value = quote(null_value)`),
// cells joined by the delimiter, '\n' after the row. f64 (ryu d2fixed, 8 digits) is not written on
// device for |v| < 2^63 (exact integer arithmetic below); larger magnitudes make the call report TPLX_E_UNSUPPORTED and the
// caller formats on the host.
TPLX_HD uint32_t csv_i64_len(int64_t v) {
    uint64_t m = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    uint32_t n = v < 0 ? 2u : 1u;
    while (m >= 10) {
        m /= 10;
        ++n;
    }
    return n;
}
TPLX_HD uint32_t csv_i64_write(uint8_t *p, int64_t v) {
    const uint32_t n = csv_i64_len(v);
    uint64_t m = v < 0 ? (uint64_t)0 - (uint64_t)v : (uint64_t)v;
    if (v < 0) p[0] = '-';
    uint32_t k = n;
    do {
        p[--k] = (uint8_t)('0' + m % 10);
        m /= 10;
    } while (m);
    return n;
}
TPLX_HD uint32_t csv_quoted_len(const uint8_t *s, uint32_t len, uint8_t delim, uint8_t quote) {
    uint32_t nq = 0;
    bool need = false;
    for (uint32_t i = 0; i < len; ++i) {
        nq += s[i] == quote;
        need |= s[i] == delim || s[i] == '\n' || s[i] == '\r';
    }
    return (nq || need) ? len + 2 + nq : len;
}
TPLX_HD uint32_t csv_quoted_write(uint8_t *p, const uint8_t *s, uint32_t len, uint8_t delim, uint8_t quote) {
    const uint32_t out = csv_quoted_len(s, len, delim, quote);
    if (out == len) {
        for (uint32_t i = 0; i < len; ++i) p[i] = s[i];
        return len;
    }
    uint32_t o = 0;
    p[o++] = quote;
    for (uint32_t i = 0; i < len; ++i) {
        if (s[i] == quote) p[o++] = quote;
        p[o++] = s[i];
    }
    p[o++] = quote;
    return o;
}

// f64 -> fixed notation with 8 decimals, correctly rounded (ties to even on the exact binary value): what the reference's
// row writer gets from ryu's d2fixed_buffered_n(d, 8, buf) (third-party ryu, not vendored in the reference tree; restated
// from its published contract = printf("%.8f") digits; special values per ryu d2fixed.c copy_special_str_printf: "nan",
// "Infinity", "-Infinity"). Exact integer arithmetic: value = m * 2^e2; the fraction m_frac * 10^8 fits in 80 bits.
// Returns the length, or 0 when |v| >= 2^63 (needs a bignum: the caller falls back to the host formatter).
TPLX_HD uint32_t csv_f64_fixed8(double v, uint8_t *out /* may be null: length only */) {
    uint64_t bits;
    bits = *reinterpret_cast<const uint64_t *>(&v);
    const bool neg = (bits >> 63) != 0;
    const uint32_t ex = (uint32_t)((bits >> 52) & 0x7FF);
    const uint64_t mant = bits & 0xFFFFFFFFFFFFFull;
    uint32_t o = 0;
    if (ex == 0x7FF) {
        const char *t = mant ? "nan" : (neg ? "-Infinity" : "Infinity");
        while (t[o]) {
            if (out) out[o] = (uint8_t)t[o];
            ++o;
        }
        return o;
    }
    const uint64_t m = ex ? (mant | (1ull << 52)) : mant;
    const int32_t e2 = (int32_t)(ex ? ex : 1) - 1075;
    uint64_t ip = 0, frac8 = 0;  // integer part, 8 fraction digits
    if (e2 >= 0) {
        if (e2 > 10) return 0;
        ip = m << e2;
    } else {
        const uint32_t k = (uint32_t)(-e2);
        if (k <= 100) {
            ip = k < 64 ? (m >> k) : 0;
            const uint64_t fr = k < 64 ? (m & ((1ull << k) - 1)) : m;
            const unsigned __int128 F = (unsigned __int128)fr * 100000000ull;
            const unsigned __int128 one = (unsigned __int128)1 << k;
            frac8 = (uint64_t)(F >> k);
            const unsigned __int128 rem = F & (one - 1), half = one >> 1;
            if (rem > half || (rem == half && (frac8 & 1))) ++frac8;
            if (frac8 == 100000000ull) {
                frac8 = 0;
                ++ip;
            }
        }  // smaller values round to zero
    }
    if (neg) {
        if (out) out[o] = '-';
        ++o;
    }
    uint32_t nd = 1;
    for (uint64_t t = ip; t >= 10; t /= 10) ++nd;
    if (out) {
        uint64_t t = ip;
        for (uint32_t i = nd; i-- > 0;) {
            out[o + i] = (uint8_t)('0' + t % 10);
            t /= 10;
        }
        out[o + nd] = '.';
        uint64_t f = frac8;
        for (uint32_t i = 8; i-- > 0;) {
            out[o + nd + 1 + i] = (uint8_t)('0' + f % 10);
            f /= 10;
        }
    }
    return o + nd + 9;
}

constexpr uint32_t CSV_NULL_CAP = 128;  // bytes of the quoted null value a None cell is written as

struct CsvSinkCols {
    uint32_t n_cols;
    uint8_t delim, quote;
    uint8_t types[TPLX_MAX_COLS];
    const uint64_t *data[TPLX_MAX_COLS];
    const uint32_t *offsets[TPLX_MAX_COLS];
    const uint8_t *bytes[TPLX_MAX_COLS];
    const uint32_t *valid[TPLX_MAX_COLS];  // Option column: validity words (a clear bit = None cell), else null
    uint32_t null_len;                     // a None cell is written as null_text[0, null_len): the null value, quoted once
    uint8_t null_text[CSV_NULL_CAP];
};
TPLX_HD bool csv_sink_is_none(const CsvSinkCols &C, uint32_t c, uint64_t r) {
    return C.valid[c] && !((C.valid[c][r >> 5] >> (r & 31)) & 1u);
}
// returns 0 when a cell cannot be formatted here (f64 of magnitude >= 2^63)
TPLX_HD uint64_t csv_sink_row_len(const CsvSinkCols &C, uint64_t r) {
    uint64_t n = C.n_cols;  // delimiters + newline
    for (uint32_t c = 0; c < C.n_cols; ++c) {
        if (csv_sink_is_none(C, c, r))
            n += C.null_len;
        else if (C.types[c] == TPLX_T_F64) {
            const uint32_t l = csv_f64_fixed8(*reinterpret_cast<const double *>(&C.data[c][r]), nullptr);
            if (!l) return 0;
            n += l;
        } else if (C.types[c] == TPLX_T_STR)
            n += csv_quoted_len(C.bytes[c] + C.offsets[c][r], C.offsets[c][r + 1] - C.offsets[c][r], C.delim, C.quote);
        else if (C.types[c] == TPLX_T_BOOL)
            n += C.data[c][r] ? 4 : 5;
        else
            n += csv_i64_len((int64_t)C.data[c][r]);
    }
    return n;
}
TPLX_HD void csv_sink_row_write(const CsvSinkCols &C, uint64_t r, uint8_t *p) {
    for (uint32_t c = 0; c < C.n_cols; ++c) {
        if (csv_sink_is_none(C, c, r)) {
            for (uint32_t k = 0; k < C.null_len; ++k) *p++ = C.null_text[k];
        } else if (C.types[c] == TPLX_T_STR)
            p += csv_quoted_write(p, C.bytes[c] + C.offsets[c][r], C.offsets[c][r + 1] - C.offsets[c][r], C.delim, C.quote);
        else if (C.types[c] == TPLX_T_F64)
            p += csv_f64_fixed8(*reinterpret_cast<const double *>(&C.data[c][r]), p);
        else if (C.types[c] == TPLX_T_BOOL) {
            const char *t = C.data[c][r] ? "true" : "false";
            while (*t) *p++ = (uint8_t)*t++;
        } else
            p += csv_i64_write(p, (int64_t)C.data[c][r]);
        *p++ = c + 1 == C.n_cols ? (uint8_t)'\n' : C.delim;
    }
}

}  // namespace tplx
