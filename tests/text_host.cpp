// Host shim over tuplex_b200/csrc/textops.cuh: K10's pipeline (text.cuh) with plain loops standing in for the grid — line
// ends by 64-byte spans over a buffer laid out like tplx_gpu_csv_upload's ('\n' at [n], zero padding), per-tile ASCII flags,
// per-line length / null / good, then the column (offsets + bytes), the validity words and the bad rows. tests/test_text_source.py
// fuzzes it against the host reader. Test infrastructure only.
#include "../tuplex_b200/csrc/textops.cuh"
#include <string.h>
#include <vector>
using namespace tplx;

static const uint32_t TILE = 256 * TEXT_SPAN;

struct HostText {
    std::vector<uint32_t> ends, offsets{0}, valid, rowmap, bad;  // bad: 4 per row (row, code, line_start, line_end)
    std::vector<uint8_t> bytes;
};

extern "C" {
HostText *htext_parse(const uint8_t *data, uint32_t n, uint32_t n_nulls, const char *const *nulls, int option) {
    HostText *H = new HostText();
    const uint64_t padded = ((uint64_t)n + 1 + TILE - 1) / TILE * TILE;
    std::vector<uint8_t> buf(padded + 64, 0);
    memcpy(buf.data(), data, n);
    buf[n] = '\n';
    std::vector<uint8_t> tile_ascii(padded / TILE, 1);
    for (uint64_t start = 0; start < padded; start += TEXT_SPAN) {
        bool ascii = true;
        text_walk_span(buf.data(), start, n, &ascii, [&](uint64_t pos) { H->ends.push_back((uint32_t)pos); });
        if (!ascii) tile_ascii[start / TILE] = 0;
    }
    CsvNulls nv{};
    nv.n = (uint8_t)n_nulls;
    uint32_t nvb = 0;
    for (uint32_t k = 0; k < n_nulls; ++k) {
        nv.off[k] = (uint8_t)nvb;
        memcpy(nv.bytes + nvb, nulls[k], strlen(nulls[k]));
        nvb += (uint32_t)strlen(nulls[k]);
    }
    nv.off[n_nulls] = (uint8_t)nvb;
    const uint32_t nl = (uint32_t)H->ends.size();
    for (uint32_t i = 0; i < nl; ++i) {
        uint32_t s, e;
        text_line_range(buf.data(), H->ends.data(), i, &s, &e);
        bool ascii = true;
        if (e > s)
            for (uint32_t t = s / TILE; t <= (e - 1) / TILE && ascii; ++t) ascii = tile_ascii[t] != 0;
        bool replaced = false;
        const uint64_t out = ascii ? (uint64_t)(e - s) : text_replaced_len(buf.data() + s, e - s, &replaced);
        const bool null = nv.n && out <= 64 && text_is_null(buf.data() + s, e - s, !replaced, out, nv);
        if (!option && null) {
            H->bad.insert(H->bad.end(), {i, 50u, i == 0 ? 0u : H->ends[i - 1] + 1, H->ends[i]});
            continue;
        }
        const uint32_t pos = (uint32_t)H->rowmap.size();
        H->rowmap.push_back(i);
        if (option && nv.n) {
            if (H->valid.size() <= pos / 32) H->valid.push_back(0);
            if (!null) H->valid[pos / 32] |= 1u << (pos & 31);
        }
        if (!null) {
            if (replaced)
                text_replaced_emit(buf.data() + s, e - s, [&](uint8_t b) { H->bytes.push_back(b); });
            else
                H->bytes.insert(H->bytes.end(), buf.begin() + s, buf.begin() + e);
        }
        H->offsets.push_back((uint32_t)H->bytes.size());
    }
    return H;
}
void htext_counts(HostText *H, uint64_t *out) {
    out[0] = H->ends.size();
    out[1] = H->rowmap.size();
    out[2] = H->bad.size() / 4;
    out[3] = H->bytes.size();
    out[4] = H->valid.size();
}
const uint32_t *htext_ends(HostText *H) { return H->ends.data(); }
const uint32_t *htext_offsets(HostText *H) { return H->offsets.data(); }
const uint8_t *htext_bytes(HostText *H) { return H->bytes.data(); }
const uint32_t *htext_valid(HostText *H) { return H->valid.data(); }
const uint32_t *htext_rowmap(HostText *H) { return H->rowmap.data(); }
const uint32_t *htext_bad(HostText *H) { return H->bad.data(); }
void htext_free(HostText *H) { delete H; }
// the replacement of one byte string: returns the replaced length, writes the bytes to out (may be null)
uint64_t htext_replace(const uint8_t *p, uint32_t len, uint8_t *out) {
    bool replaced = false;
    const uint64_t l = text_replaced_len(p, len, &replaced);
    if (out) {
        uint64_t w = 0;
        text_replaced_emit(p, len, [&](uint8_t b) { out[w++] = b; });
    }
    return l;
}
// k pieces of w bytes, `stride` apart in p: each replaced on its own (its end is a line end), written to out followed by sep
uint64_t htext_replace_pieces(const uint8_t *p, uint64_t k, uint32_t w, uint32_t stride, uint8_t sep, uint8_t *out) {
    uint64_t o = 0;
    for (uint64_t i = 0; i < k; ++i) {
        text_replaced_emit(p + i * stride, w, [&](uint8_t b) { out[o++] = b; });
        out[o++] = sep;
    }
    return o;
}
}
