// Host shim over tuplex_b200/csrc/csvops.cuh for Option[T] columns: the per-row parse the CUDA kernels run
// (csv_parse_one_row with its null mask), with the sequential row finder and a plain loop standing in for the grid, then
// the compaction and the validity words csv_pack_valid builds (block row order, bit r & 31 of word r >> 5 set = present).
// tests/test_csv_option.py fuzzes it against a reference built on the C oracle. Test infrastructure only.
#include "../tuplex_b200/csrc/csvops.cuh"
#include <string.h>
#include <vector>
using namespace tplx;

struct HostOptCsv {
    uint32_t n_out = 0, n_rows = 0, n_good = 0;
    uint8_t out_types[TPLX_MAX_COLS];
    std::vector<uint64_t> fixed[TPLX_MAX_COLS];
    std::vector<uint32_t> offsets[TPLX_MAX_COLS];
    std::vector<uint8_t> bytes[TPLX_MAX_COLS];
    std::vector<uint32_t> valid[TPLX_MAX_COLS];  // empty for a column that is not Option
    std::vector<uint32_t> rowmap, bad;           // bad: 4 per row (row, code, line_start, line_end)
};

extern "C" {
HostOptCsv *hopt_parse(const uint8_t *data, uint32_t n, uint8_t delim, uint8_t quote, int skip_header, uint32_t n_file_cols,
                       const uint8_t *col_types, uint32_t n_nulls, const char *const *nulls) {
    HostOptCsv *H = new HostOptCsv();
    std::vector<uint8_t> buf((size_t)n + 128, 0);
    memcpy(buf.data(), data, n);
    buf[n] = '\n';
    std::vector<uint32_t> row_end((size_t)n / 2 + 2, 0);
    const uint32_t total = csv_find_rows_sequential(buf.data(), n, delim, quote, row_end.data());
    CsvParseParams P{};
    std::vector<uint8_t> kind(col_types, col_types + n_file_cols), slot(n_file_cols, 0);
    bool any_option = false;
    for (uint32_t c = 0; c < n_file_cols; ++c) {
        if (kind[c] == CSV_SKIP) continue;
        const uint8_t t = kind[c] & ~TPLX_T_OPTION;
        any_option |= (kind[c] & TPLX_T_OPTION) != 0;
        slot[c] = (uint8_t)P.n_out;
        P.out_types[P.n_out] = t;
        P.strk[P.n_out] = t == TPLX_T_STR ? (int8_t)P.n_str++ : (int8_t)-1;
        ++P.n_out;
    }
    P.nulls.n = (uint8_t)n_nulls;
    uint32_t nvb = 0;
    for (uint32_t k = 0; k < n_nulls; ++k) {
        P.nulls.off[k] = (uint8_t)nvb;
        memcpy(P.nulls.bytes + nvb, nulls[k], strlen(nulls[k]));
        nvb += (uint32_t)strlen(nulls[k]);
    }
    P.nulls.off[n_nulls] = (uint8_t)nvb;
    P.r0 = skip_header ? 1 : 0;
    const uint32_t nd = total > P.r0 ? total - P.r0 : 0;
    std::vector<uint64_t> tmp[TPLX_MAX_COLS], lens((size_t)(P.n_str ? P.n_str : 1) * (nd + 1), 0), good(nd + 1, 0), mask(nd + 1, 0);
    std::vector<uint32_t> code(nd + 1, 0);
    uint32_t flags[4] = {0, 0, 0, 0};
    P.buf = buf.data();
    P.n = n;
    P.row_end = row_end.data();
    P.nd = nd;
    P.delim = delim;
    P.quote = quote;
    P.n_file_cols = n_file_cols;
    P.col_kind = kind.data();
    P.col_slot = slot.data();
    P.flags = flags;
    for (uint32_t c = 0; c < P.n_out; ++c) {
        tmp[c].assign(nd + 1, 0);
        P.tmp[c] = tmp[c].data();
    }
    P.lens = lens.data();
    P.good = good.data();
    P.code = code.data();
    P.nullmask = any_option ? mask.data() : nullptr;
    for (uint32_t i = 0; i < nd; ++i) csv_parse_one_row(P, i);
    H->n_out = P.n_out;
    H->n_rows = nd;
    memcpy(H->out_types, P.out_types, sizeof H->out_types);
    for (uint32_t c = 0; c < P.n_out; ++c)
        if (P.out_types[c] == TPLX_T_STR) H->offsets[c].push_back(0);
    std::vector<uint8_t> is_opt(P.n_out, 0);
    for (uint32_t c = 0; c < n_file_cols; ++c)
        if (kind[c] != CSV_SKIP && (kind[c] & TPLX_T_OPTION)) is_opt[slot[c]] = 1;
    for (uint32_t i = 0; i < nd; ++i) {
        if (code[i]) {
            const uint32_t r = P.r0 + i;
            H->bad.insert(H->bad.end(), {i, code[i], csv_row_start(buf.data(), row_end.data(), r), row_end[r]});
            continue;
        }
        const uint32_t pos = H->n_good++;
        H->rowmap.push_back(i);
        for (uint32_t c = 0; c < P.n_out; ++c) {
            if (is_opt[c]) {
                if (H->valid[c].size() <= pos / 32) H->valid[c].push_back(0);
                if (!((mask[i] >> c) & 1)) H->valid[c][pos / 32] |= 1u << (pos & 31);
            }
            if (P.out_types[c] != TPLX_T_STR) {
                H->fixed[c].push_back(tmp[c][i]);
                continue;
            }
            const uint64_t info = tmp[c][i];
            const uint32_t b = (uint32_t)info, raw = (uint32_t)(info >> 32) & 0x7FFFFFFFu;
            std::vector<uint8_t> t(raw + 1);
            const uint32_t l = csv_dequote(buf.data(), b, b + raw, (info >> 63) ? quote : (uint8_t)0, t.data(), raw + 1);
            H->bytes[c].insert(H->bytes[c].end(), t.begin(), t.begin() + l);
            H->offsets[c].push_back((uint32_t)H->bytes[c].size());
        }
    }
    return H;
}
void hopt_counts(HostOptCsv *H, uint32_t *out) { out[0] = H->n_out; out[1] = H->n_rows; out[2] = H->n_good; out[3] = (uint32_t)(H->bad.size() / 4); }
uint32_t hopt_type(HostOptCsv *H, uint32_t c) { return H->out_types[c]; }
const uint64_t *hopt_fixed(HostOptCsv *H, uint32_t c) { return H->fixed[c].data(); }
const uint32_t *hopt_offsets(HostOptCsv *H, uint32_t c) { return H->offsets[c].data(); }
const uint8_t *hopt_bytes(HostOptCsv *H, uint32_t c, uint64_t *n) { *n = H->bytes[c].size(); return H->bytes[c].data(); }
const uint32_t *hopt_valid(HostOptCsv *H, uint32_t c, uint32_t *n) { *n = (uint32_t)H->valid[c].size(); return H->valid[c].data(); }
const uint32_t *hopt_rowmap(HostOptCsv *H) { return H->rowmap.data(); }
const uint32_t *hopt_bad(HostOptCsv *H) { return H->bad.data(); }
void hopt_free(HostOptCsv *H) { delete H; }
// K7 with None cells: the device row writer over host column arrays and validity words
unsigned long long hopt_write(unsigned n_cols, const uint8_t *types, const uint64_t *const *data, const uint32_t *const *offsets,
                              const uint8_t *const *bytes, const uint32_t *const *valid, unsigned long long n_rows, uint8_t delim,
                              uint8_t quote, const char *null_value, uint8_t *out) {
    CsvSinkCols C{};
    C.n_cols = n_cols;
    C.delim = delim;
    C.quote = quote;
    C.null_len = csv_quoted_write(C.null_text, (const uint8_t *)null_value, (uint32_t)strlen(null_value), delim, quote);
    for (unsigned c = 0; c < n_cols; ++c) {
        C.types[c] = types[c];
        C.data[c] = data[c];
        C.offsets[c] = offsets[c];
        C.bytes[c] = bytes[c];
        C.valid[c] = valid[c];
    }
    unsigned long long pos = 0;
    for (unsigned long long r = 0; r < n_rows; ++r) {
        const uint64_t l = csv_sink_row_len(C, r);
        if (out) csv_sink_row_write(C, r, out + pos);
        pos += l;
    }
    return pos;
}
}
