// textops.cuh — per-line semantics of K10 (text file -> one string column), shared by the kernels (text.cuh) and by host
// builds (tests/text_host.cpp): the line-end test over a word, the '\r' trim, UTF-8 validation with CPython's replacement,
// and the match against the null values.
//
// The contract is Context.text's host reader (tuplex_b200/textsource.py, `read_lines`): lines end at '\n'; the last line
// counts without one; one trailing '\r' is stripped; an invalid line is stored as bytes.decode("utf-8", "replace").encode(),
// one U+FFFD per maximal invalid subpart; a line equal to a null value (after the strip and the replacement) is null.
// Departures from the reference's TextReader.cc (core/src/physical/TextReader.cc:60-140), all three on purpose:
//   * a lone '\r' at EOF is stripped like every other trailing '\r' (the reference keeps it);
//   * a NUL byte is content and never hides a newline (the reference's _mm_cmpistri compare is implicit-length, so a NUL
//     ends its 16-byte window early and can merge two lines);
//   * invalid UTF-8 is replaced (the reference keeps the raw bytes).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "csvops.cuh"

namespace tplx {

constexpr uint32_t TEXT_SPAN = 64;  // bytes walked by one thread

// bit i set = byte i of the little-endian word w is '\n'
TPLX_HD uint32_t text_nl_bits(uint64_t w) { return csv_pack8(csv_eq8(w, '\n')); }
TPLX_HD bool text_word_ascii(uint64_t w) { return (w & 0x8080808080808080ull) == 0; }

TPLX_HD uint32_t text_popc(uint32_t x) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

// Line ends inside the span [start, start + TEXT_SPAN) of a buffer of n data bytes followed by '\n' at [n] and zero padding
// (tplx_gpu_csv_upload): every '\n' before n, and n itself when the data does not end with '\n' (the last line has no
// newline of its own). The appended '\n' after a final '\n', or after no data, makes no line. emit(pos) is called for each
// line end in order; returns their number. *ascii is cleared when the span holds a byte >= 0x80.
template <class Emit>
TPLX_HD uint32_t text_walk_span(const uint8_t *buf, uint64_t start, uint64_t n, bool *ascii, Emit &&emit) {
    uint32_t cnt = 0;
    const bool tail_line = n > 0 && buf[n - 1] != '\n';
    for (uint32_t k = 0; k < TEXT_SPAN / 8; ++k) {
        const uint64_t p0 = start + 8 * k;
        const uint64_t w = csv_load8(buf + p0);
        uint32_t nl = text_nl_bits(w);
        if (p0 <= n && n < p0 + 8 && !tail_line) nl &= ~(1u << (uint32_t)(n - p0));
        if (!text_word_ascii(w)) *ascii = false;
        cnt += text_popc(nl);
        while (nl) {
            const uint32_t i = csv_ctz64(nl);
            emit(p0 + i);
            nl &= nl - 1;
        }
    }
    return cnt;
}

// [*s, *e) = bytes of line i without its newline and without one trailing '\r'; ends[i] = position of the newline ending line i
TPLX_HD void text_line_range(const uint8_t *buf, const uint32_t *ends, uint32_t i, uint32_t *s, uint32_t *e) {
    const uint32_t b = i == 0 ? 0u : ends[i - 1] + 1;
    uint32_t x = ends[i];
    if (x > b && buf[x - 1] == '\r') --x;
    *s = b;
    *e = x;
}

// One step of CPython's UTF-8 decoder over p[0..len), len >= 1 (Objects/stringlib/codecs.h; the Unicode standard's maximal
// subpart practice): returns the bytes consumed; *ok = they form one valid character (kept as they are), else they are one
// maximal invalid subpart (one U+FFFD).
TPLX_HD uint32_t text_utf8_step(const uint8_t *p, uint32_t len, bool *ok) {
    const uint8_t c = p[0];
    *ok = true;
    if (c < 0x80) return 1;
    uint32_t need;
    uint8_t lo = 0x80, hi = 0xBF;
    if (c >= 0xC2 && c <= 0xDF) {
        need = 1;
    } else if (c >= 0xE0 && c <= 0xEF) {
        need = 2;
        if (c == 0xE0) lo = 0xA0;
        if (c == 0xED) hi = 0x9F;
    } else if (c >= 0xF0 && c <= 0xF4) {
        need = 3;
        if (c == 0xF0) lo = 0x90;
        if (c == 0xF4) hi = 0x8F;
    } else {
        *ok = false;
        return 1;
    }
    for (uint32_t k = 1; k <= need; ++k) {
        if (k >= len || p[k] < lo || p[k] > hi) {
            *ok = false;
            return k;
        }
        lo = 0x80;
        hi = 0xBF;
    }
    return need + 1;
}

// bytes of p[0..len) after the replacement; *replaced = some subpart was invalid (else the line is kept verbatim)
TPLX_HD uint64_t text_replaced_len(const uint8_t *p, uint32_t len, bool *replaced) {
    uint64_t o = 0;
    bool r = false;
    for (uint32_t k = 0; k < len;) {
        bool ok;
        const uint32_t m = text_utf8_step(p + k, len - k, &ok);
        o += ok ? m : 3;
        r = r || !ok;
        k += m;
    }
    *replaced = r;
    return o;
}

// out(byte) for every byte of p[0..len) after the replacement, in order
template <class Out>
TPLX_HD void text_replaced_emit(const uint8_t *p, uint32_t len, Out &&out) {
    for (uint32_t k = 0; k < len;) {
        bool ok;
        const uint32_t m = text_utf8_step(p + k, len - k, &ok);
        if (ok) {
            for (uint32_t j = 0; j < m; ++j) out(p[k + j]);
        } else {
            out(0xEF);
            out(0xBF);
            out(0xBD);
        }
        k += m;
    }
}

// Is the line p[0..len) (out_len bytes after the replacement; verbatim = nothing in it is replaced) a null value?
TPLX_HD bool text_is_null(const uint8_t *p, uint32_t len, bool verbatim, uint64_t out_len, const CsvNulls &nv) {
    for (uint32_t k = 0; k < nv.n; ++k) {
        const uint8_t *v = nv.bytes + nv.off[k];
        const uint32_t vl = (uint32_t)(nv.off[k + 1] - nv.off[k]);
        if (vl != out_len) continue;
        bool eq = true;
        if (verbatim) {
            for (uint32_t j = 0; j < vl && eq; ++j) eq = p[j] == v[j];
        } else {
            uint32_t o = 0;
            text_replaced_emit(p, len, [&](uint8_t b) { eq = eq && b == v[o++]; });
        }
        if (eq) return true;
    }
    return false;
}

}  // namespace tplx
