// host.cu — the C ABI (include/frz_cuda.h): host-side mirror of the reference's Matcher / Pattern /
// Config logic for the match_list path, orchestrating the CUDA stages.  No CPU compute fallback.
//
// Reference logic mirrored here (file:line relative to the reference crate):
//   Pattern::parse / parse_query          src/pattern.rs:100-222
//   PatternConfig::resolve                src/pattern.rs:250-262
//   Matcher::build_patterns / compile     src/matcher/mod.rs:178-205
//   Matcher::get_backend                  src/matcher/mod.rs:448-498
//   score_fits_in_u8                      src/smith_waterman/mod.rs:91-116
//   Scoring::guard_against_score_overflow src/lib.rs:506-537
//   Matcher::match_list / match_list_into src/matcher/mod.rs:212-222, 373-392
//   match_list_multi_into                 src/matcher/multi.rs:84-152
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <mutex>

#include "frz_device.cuh"
#include "frz_host.h"
#include "unicode_needle.h"
#include "indices_path.cuh"

// ------------------------------------------------------------------------------------ errors

static thread_local char g_err[512] = "";

frz_status frz_fail(frz_status s, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return s;
}

extern "C" const char* frz_last_error(void) { return g_err; }
extern "C" int frz_abi_version(void) { return FRZ_ABI_VERSION; }
extern "C" const char* frz_status_str(frz_status s) {
    switch (s) {
        case FRZ_OK: return "ok";
        case FRZ_ERR_INVALID_ARG: return "invalid argument";
        case FRZ_ERR_NEEDLE_TOO_LONG: return "needle too long and could overflow the u16 score";
        case FRZ_ERR_GAP_OVERFLOW: return "gap penalties too large and could overflow the u16 score";
        case FRZ_ERR_TOO_MANY_ITEMS: return "too many items in haystack, will overflow the u32 index";
        case FRZ_ERR_THREADS_ZERO: return "threads must be positive";
        case FRZ_ERR_CAPACITY: return "output capacity too small";
        case FRZ_ERR_CUDA: return "CUDA error";
        case FRZ_ERR_NO_DEVICE: return "no usable CUDA device";
        case FRZ_ERR_UNSUPPORTED: return "not supported on the GPU path";
        case FRZ_ERR_OOM: return "out of device memory";
        case FRZ_ERR_NCCL: return "NCCL error";
    }
    return "?";
}

extern "C" void frz_scoring_default(frz_scoring* s) {
    *s = frz_scoring{12, 6, 5, 1, 12, 4, 4, 8, 4};  // src/const.rs:1-10
}
extern "C" void frz_config_default(frz_config* c) {
    memset(c, 0, sizeof *c);
    c->max_typos = 0;
    c->casing = FRZ_CASE_SMART;
    c->unicode = FRZ_UNICODE_SMART;
    c->matching = FRZ_MATCHING_FUZZY;
    c->sort = FRZ_SORT_SCORE_THEN_INDEX_ASC;
    frz_scoring_default(&c->scoring);
    c->emulate_lanes = 0;
}

frz_status frz_ensure_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return frz_fail(FRZ_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU fallback",
                        e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= n) return frz_fail(FRZ_ERR_INVALID_ARG, "device %d out of range (have %d)", device, n);
    FRZ_CUDA_TRY(cudaSetDevice(device));
    return FRZ_OK;
}

frz_status frz_check_offset_width(int offset_width) {
    if (offset_width != 4 && offset_width != 8) return frz_fail(FRZ_ERR_INVALID_ARG, "offset_width must be 4 or 8");
    return FRZ_OK;
}

// Matcher::guard_against_haystack_overflow (src/matcher/mod.rs:438-446)
frz_status frz_check_index_range(uint64_t n, uint32_t index_offset) {
    if (n + index_offset > 0xFFFFFFFFull)
        return frz_fail(FRZ_ERR_TOO_MANY_ITEMS, "too many items in haystack, will overflow the u32 index: %llu > %u (index offset: %u)",
                        (unsigned long long)(n + index_offset), 0xFFFFFFFFu, index_offset);
    return FRZ_OK;
}

// ----------------------------------------------------------------------------- query parser

struct OwnedPattern {
    std::string needle;
    std::string raw;
    bool negated = false;
    int matching = -1, casing = -1, unicode = -1, max_typos = -1;
    bool has_scoring = false;
    frz_scoring scoring{};
};

struct frz_query {
    std::vector<OwnedPattern> pats;
};

namespace {

// Decodes one UTF-8 scalar starting at s[i] (input is a Rust &str, so valid UTF-8; be lenient).
uint32_t utf8_next(const uint8_t* s, size_t len, size_t* i) {
    uint8_t b = s[*i];
    int extra = b < 0x80 ? 0 : (b >> 5) == 6 ? 1 : (b >> 4) == 14 ? 2 : (b >> 3) == 30 ? 3 : 0;
    uint32_t cp = extra == 0 ? b : extra == 1 ? (b & 0x1f) : extra == 2 ? (b & 0x0f) : (b & 0x07);
    size_t j = *i + 1;
    for (int k = 0; k < extra && j < len; k++, j++) cp = (cp << 6) | (s[j] & 0x3f);
    *i = j;
    return cp;
}
void utf8_push(std::string& out, uint32_t cp) {
    if (cp < 0x80) out.push_back((char)cp);
    else if (cp < 0x800) { out.push_back((char)(0xC0 | (cp >> 6))); out.push_back((char)(0x80 | (cp & 0x3f))); }
    else if (cp < 0x10000) {
        out.push_back((char)(0xE0 | (cp >> 12))); out.push_back((char)(0x80 | ((cp >> 6) & 0x3f))); out.push_back((char)(0x80 | (cp & 0x3f)));
    } else {
        out.push_back((char)(0xF0 | (cp >> 18))); out.push_back((char)(0x80 | ((cp >> 12) & 0x3f)));
        out.push_back((char)(0x80 | ((cp >> 6) & 0x3f))); out.push_back((char)(0x80 | (cp & 0x3f)));
    }
}
// char::is_whitespace (Unicode White_Space)
bool is_ws(uint32_t c) {
    return (c >= 9 && c <= 13) || c == 0x20 || c == 0x85 || c == 0xA0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200A) ||
           c == 0x2028 || c == 0x2029 || c == 0x202F || c == 0x205F || c == 0x3000;
}

// Pattern::parse (src/pattern.rs:100-165)
OwnedPattern parse_atom(const uint8_t* atom, size_t len) {
    struct Tok { uint32_t c; bool escaped; };
    std::vector<Tok> toks;
    size_t i = 0;
    while (i < len) {
        uint32_t c = utf8_next(atom, len, &i);
        if (c == '\\' && i < len) toks.push_back({utf8_next(atom, len, &i), true});
        else toks.push_back({c, false});
    }
    size_t lo = 0, hi = toks.size();
    auto strip_first = [&](uint32_t op) {
        if (lo < hi && !toks[lo].escaped && toks[lo].c == op) { lo++; return true; }
        return false;
    };
    auto strip_last = [&](uint32_t op) {
        if (lo < hi && !toks[hi - 1].escaped && toks[hi - 1].c == op) { hi--; return true; }
        return false;
    };
    OwnedPattern p;
    p.raw.assign((const char*)atom, len);
    p.negated = strip_first('!');
    bool prefix = strip_first('^');
    bool substring = !prefix && strip_first('\'');
    bool suffix = strip_last('$');
    auto is_special = [](uint32_t c) { return c == '!' || c == '^' || c == '\'' || c == '$' || is_ws(c); };
    for (size_t k = lo; k < hi; k++) {
        if (toks[k].escaped && !is_special(toks[k].c)) p.needle.push_back('\\');
        utf8_push(p.needle, toks[k].c);
    }
    if (prefix && suffix) p.matching = FRZ_MATCHING_EXACT;
    else if (prefix) p.matching = FRZ_MATCHING_PREFIX;
    else if (suffix) p.matching = FRZ_MATCHING_SUFFIX;
    else if (substring) p.matching = FRZ_MATCHING_SUBSTRING;
    else if (p.negated) p.matching = FRZ_MATCHING_SUBSTRING;
    else p.matching = -1;
    return p;
}

// Pattern::parse_query (src/pattern.rs:190-222)
std::vector<OwnedPattern> parse_query(const uint8_t* q, size_t len) {
    std::vector<OwnedPattern> out;
    bool have_start = false, escaped = false;
    size_t start = 0;
    auto push = [&](size_t a, size_t b) {
        OwnedPattern p = parse_atom(q + a, b - a);
        if (!p.needle.empty()) out.push_back(std::move(p));
    };
    size_t i = 0;
    while (i < len) {
        size_t at = i;
        uint32_t c = utf8_next(q, len, &i);
        if (escaped) escaped = false;
        else if (c == '\\') { if (!have_start) { have_start = true; start = at; } escaped = true; }
        else if (is_ws(c)) { if (have_start) { push(start, at); have_start = false; } }
        else if (!have_start) { have_start = true; start = at; }
    }
    if (have_start) push(start, len);
    return out;
}

void fill_c_pattern(const OwnedPattern& o, frz_pattern* out) {
    memset(out, 0, sizeof *out);
    out->needle = (const uint8_t*)o.needle.data();
    out->needle_len = o.needle.size();
    out->negated = o.negated;
    out->has_scoring = o.has_scoring;
    out->casing = (int8_t)o.casing;
    out->unicode = (int8_t)o.unicode;
    out->matching = (int8_t)o.matching;
    out->max_typos = o.max_typos;
    out->scoring = o.scoring;
}

}  // namespace

extern "C" frz_status frz_parse_query(const uint8_t* query, size_t len, frz_query** out) {
    if (!out || (!query && len)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    auto* q = new frz_query();
    q->pats = parse_query(query, len);
    *out = q;
    return FRZ_OK;
}
extern "C" frz_status frz_parse_atom(const uint8_t* atom, size_t len, frz_query** out) {
    if (!out || (!atom && len)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    auto* q = new frz_query();
    q->pats.push_back(parse_atom(atom, len));
    *out = q;
    return FRZ_OK;
}
extern "C" size_t frz_query_len(const frz_query* q) { return q ? q->pats.size() : 0; }
extern "C" frz_status frz_query_get(const frz_query* q, size_t i, frz_pattern* out) {
    if (!q || !out || i >= q->pats.size()) return frz_fail(FRZ_ERR_INVALID_ARG, "pattern index out of range");
    fill_c_pattern(q->pats[i], out);
    return FRZ_OK;
}
extern "C" void frz_query_destroy(frz_query* q) { delete q; }

// ---------------------------------------------------------------------------------- corpus

extern "C" frz_status frz_corpus_create_device(const uint8_t* d_bytes, const uint64_t* d_offsets, uint64_t n,
                                               uint64_t total_bytes, int device, void* stream, frz_corpus** out) {
    if (!out) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    if (n > 0xFFFFFFFFull) return frz_fail(FRZ_ERR_TOO_MANY_ITEMS, "too many items in haystack: %llu", (unsigned long long)n);
    FRZ_TRY(frz_ensure_device(device));
    auto c = std::make_unique<frz_corpus>();
    c->st.device = device;
    frz_status s = frz_pack_corpus_device(d_bytes, d_offsets, 8, n, total_bytes, (cudaStream_t)stream, &c->st);
    // the corpus is complete on return: matches run on other streams, and the caller may free the inputs
    if (s == FRZ_OK && cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess)
        s = frz_fail(FRZ_ERR_CUDA, "pack failed: %s", cudaGetErrorString(cudaGetLastError()));
    if (s != FRZ_OK) return s;
    *out = c.release();
    return FRZ_OK;
}

// Host Arrow buffers (Utf8: 32-bit offsets, LargeUtf8: 64-bit; a sliced array may start at offsets[0] != 0).
extern "C" frz_status frz_corpus_create_arrow(const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n, int device,
                                              frz_corpus** out) {
    if (!out || !offsets) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_check_offset_width(offset_width));
    if (n > 0xFFFFFFFFull) return frz_fail(FRZ_ERR_TOO_MANY_ITEMS, "too many items in haystack: %llu", (unsigned long long)n);
    FRZ_TRY(frz_ensure_device(device));
    auto c = std::make_unique<frz_corpus>();
    c->st.device = device;
    FrzIngest ing;
    cudaStream_t stream = nullptr;
    frz_status s = frz_ingest_host(ing, bytes, offsets, offset_width, n, stream, &c->st);
    if (s == FRZ_OK && cudaStreamSynchronize(stream) != cudaSuccess)
        s = frz_fail(FRZ_ERR_CUDA, "pack failed: %s", cudaGetErrorString(cudaGetLastError()));
    if (s != FRZ_OK) return s;
    *out = c.release();
    return FRZ_OK;
}

extern "C" frz_status frz_corpus_create(const uint8_t* bytes, const uint64_t* offsets, uint64_t n, int device, frz_corpus** out) {
    return frz_corpus_create_arrow(bytes, offsets, 8, n, device, out);
}

// Incremental ingestion: the new haystacks get indices [len, len + n_new).  Synchronous; must not overlap a match
// call on the same corpus.
extern "C" frz_status frz_corpus_append(frz_corpus* c, const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n_new) {
    if (!c || (n_new && !offsets)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_check_offset_width(offset_width));
    if (n_new == 0) return FRZ_OK;
    FRZ_TRY(frz_ensure_device(c->st.device));
    if (!c->ingest) c->ingest = std::make_unique<FrzIngest>();
    cudaStream_t stream = nullptr;
    FRZ_TRY(frz_append_host(*c->ingest, bytes, offsets, offset_width, n_new, stream, &c->st));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    return FRZ_OK;
}

// In-place edits.  Every check runs on the host before anything changes, so a refused call leaves the corpus as it was.
static frz_status check_indices(const frz_corpus* c, const uint32_t* which, uint64_t n) {
    for (uint64_t j = 0; j < n; j++)
        if (which[j] >= c->st.n)
            return frz_fail(FRZ_ERR_INVALID_ARG, "index %u out of range (the corpus has %llu haystacks)", which[j],
                            (unsigned long long)c->st.n);
    return FRZ_OK;
}

extern "C" frz_status frz_corpus_remove(frz_corpus* c, const uint32_t* which, uint64_t n) {
    if (!c || (n && !which)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (n == 0) return FRZ_OK;
    FRZ_TRY(check_indices(c, which, n));
    FRZ_TRY(frz_ensure_device(c->st.device));
    if (!c->ingest) c->ingest = std::make_unique<FrzIngest>();
    return frz_remove_host(*c->ingest, which, n, nullptr, &c->st);
}

template <typename OffT>
static frz_status check_replacement_lengths(const OffT* off, uint64_t n) {
    for (uint64_t j = 0; j < n; j++) {
        if (off[j + 1] < off[j]) return frz_fail(FRZ_ERR_INVALID_ARG, "offsets decrease at %llu", (unsigned long long)j);
        if ((uint64_t)off[j + 1] - (uint64_t)off[j] > FRZ_MAX_HAY_LEN)
            return frz_fail(FRZ_ERR_UNSUPPORTED, "haystack longer than %u bytes", FRZ_MAX_HAY_LEN);
    }
    return FRZ_OK;
}

extern "C" frz_status frz_corpus_replace(frz_corpus* c, const uint32_t* which, uint64_t n, const uint8_t* bytes, const void* offsets,
                                         int offset_width) {
    if (!c || (n && (!which || !offsets))) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_check_offset_width(offset_width));
    if (n == 0) return FRZ_OK;
    FRZ_TRY(check_indices(c, which, n));
    std::vector<uint32_t> sorted(which, which + n);
    std::sort(sorted.begin(), sorted.end());
    for (uint64_t j = 1; j < n; j++)
        if (sorted[j] == sorted[j - 1]) return frz_fail(FRZ_ERR_INVALID_ARG, "index %u is replaced twice", sorted[j]);
    if (offset_width == 4) FRZ_TRY(check_replacement_lengths(static_cast<const uint32_t*>(offsets), n));
    else FRZ_TRY(check_replacement_lengths(static_cast<const uint64_t*>(offsets), n));
    const uint64_t r_bytes = offset_width == 4 ? (uint64_t)(static_cast<const uint32_t*>(offsets)[n] - static_cast<const uint32_t*>(offsets)[0])
                                               : static_cast<const uint64_t*>(offsets)[n] - static_cast<const uint64_t*>(offsets)[0];
    if (r_bytes && !bytes) return frz_fail(FRZ_ERR_INVALID_ARG, "null bytes");
    FRZ_TRY(frz_ensure_device(c->st.device));
    if (!c->ingest) c->ingest = std::make_unique<FrzIngest>();
    if (!c->edit_tiles) c->edit_tiles = std::make_unique<FrzCorpusStorage>();
    const frz_status s = frz_replace_host(*c->ingest, *c->edit_tiles, which, n, bytes, offsets, offset_width, nullptr, &c->st);
    // The staging of a replace (the touched tiles' raw bytes and metadata) is kept for the next edit while it is small; a
    // large one, up to a second copy of the list when every tile was touched, is given back at once.
    constexpr uint64_t kKeepStaging = 64ull << 20;
    FrzIngest& ing = *c->ingest;
    if (ing.d_bytes.cap() + ing.d_offsets.cap() > kKeepStaging) {
        ing.d_bytes.reset();
        ing.d_offsets.reset();
    }
    const FrzCorpusStorage& et = *c->edit_tiles;
    const uint64_t et_bytes = et.tile_base.cap() * (8 + FRZ_GROUPS_PER_TILE * sizeof(FrzGroupDesc) + FRZ_TILE * (4 + 2 + 8) + 8);
    if (et_bytes > kKeepStaging) c->edit_tiles.reset();
    return s;
}

extern "C" frz_status frz_corpus_create_ptrs(const uint8_t* const* ptrs, const uint32_t* lens, uint64_t n, int device,
                                             frz_corpus** out) {
    if (!out || (n && (!ptrs || !lens))) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    std::vector<uint64_t> off(n + 1, 0);
    for (uint64_t i = 0; i < n; i++) off[i + 1] = off[i] + lens[i];
    std::vector<uint8_t> bytes(off[n] ? off[n] : 1);
    for (uint64_t i = 0; i < n; i++)
        if (lens[i]) memcpy(bytes.data() + off[i], ptrs[i], lens[i]);
    return frz_corpus_create(bytes.data(), off.data(), n, device, out);
}

extern "C" uint64_t frz_corpus_len(const frz_corpus* c) { return c ? c->st.n : 0; }
extern "C" uint64_t frz_corpus_total_bytes(const frz_corpus* c) { return c ? c->st.total_bytes : 0; }
extern "C" uint64_t frz_corpus_device_bytes(const frz_corpus* c) {
    if (!c) return 0;
    const auto& s = c->st;
    return (s.total_units + 1) * 16 + (uint64_t)s.n_tiles * (8 + FRZ_GROUPS_PER_TILE * 16 + FRZ_TILE * (6 + 8));
}
extern "C" int frz_corpus_device(const frz_corpus* c) { return c ? c->st.device : -1; }

// Test aid: the packed image (frz_device.cuh), so that tests can check the layout against a restatement of DESIGN.md §3.
extern "C" frz_status frz_corpus_debug_image(const frz_corpus* c, void* tile_base, void* groups, void* slot_meta, void* slot_of,
                                             void* slot_sig, void* units, uint64_t sizes[6]) {
    if (!c || !sizes) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    const FrzCorpusStorage& s = c->st;
    const uint64_t slots = (uint64_t)s.n_tiles * FRZ_TILE;
    const uint64_t need[6] = {(uint64_t)s.n_tiles * sizeof(uint64_t), (uint64_t)s.n_tiles * FRZ_GROUPS_PER_TILE * sizeof(FrzGroupDesc),
                              slots * sizeof(uint32_t), slots * sizeof(uint16_t), slots * sizeof(uint2), s.total_units * sizeof(uint4)};
    const void* src[6] = {s.tile_base.get(), s.groups.get(), s.slot_meta.get(), s.slot_of.get(), s.slot_sig.get(), s.data.get()};
    void* dst[6] = {tile_base, groups, slot_meta, slot_of, slot_sig, units};
    int given = 0;
    for (void* d : dst) given += d != nullptr;
    if (given == 0) {   // size query
        memcpy(sizes, need, sizeof need);
        return FRZ_OK;
    }
    if (given != 6) return frz_fail(FRZ_ERR_INVALID_ARG, "pass all six buffers, or none for a size query");
    for (int i = 0; i < 6; i++)
        if (sizes[i] != need[i])
            return frz_fail(FRZ_ERR_INVALID_ARG, "buffer %d holds %llu bytes, the image needs %llu", i, (unsigned long long)sizes[i],
                            (unsigned long long)need[i]);
    FRZ_TRY(frz_ensure_device(s.device));
    for (int i = 0; i < 6; i++)
        if (need[i]) FRZ_CUDA_TRY(cudaMemcpy(dst[i], src[i], need[i], cudaMemcpyDeviceToHost));
    return FRZ_OK;
}
extern "C" void frz_corpus_destroy(frz_corpus* c) { delete c; }

// --------------------------------------------------------------------------------- matcher

namespace {

struct CpuIsa {
    bool avx512_pf, avx512_sw, avx512_sw_u8, avx2, sse;
};
CpuIsa detect_isa() {
    CpuIsa r{false, false, false, false, false};
#if defined(__x86_64__)
    __builtin_cpu_init();
    bool f = __builtin_cpu_supports("avx512f"), bw = __builtin_cpu_supports("avx512bw");
    bool bmi1 = __builtin_cpu_supports("bmi"), bmi2 = __builtin_cpu_supports("bmi2");
    bool vbmi = __builtin_cpu_supports("avx512vbmi");
    r.avx512_pf = f && bw && bmi1 && bmi2;       // src/prefilter/backend/avx512.rs:14-19
    r.avx512_sw = f && bw;                       // src/smith_waterman/backend/avx512.rs:44-46
    r.avx512_sw_u8 = f && bw && vbmi;            // src/smith_waterman/backend/avx512.rs:112-116
    r.avx2 = __builtin_cpu_supports("avx2");
    r.sse = __builtin_cpu_supports("sse2") && __builtin_cpu_supports("ssse3") && __builtin_cpu_supports("sse4.1");
#endif
    return r;
}

uint16_t sat_add16(uint32_t a, uint32_t b) { uint32_t r = a + b; return (uint16_t)(r > 0xFFFF ? 0xFFFF : r); }
uint16_t sat_sub16(uint32_t a, uint32_t b) { return (uint16_t)(a > b ? a - b : 0); }

uint32_t max_per_char_bonus(const frz_scoring& s) {  // src/lib.rs:488-494
    uint32_t bonus = std::max(s.delimiter_bonus, s.capitalization_bonus);
    uint32_t amort = std::max((bonus + 1) / 2, bonus > s.gap_open_penalty ? bonus - s.gap_open_penalty : 0u);
    return sat_add16(amort, s.matching_case_bonus);
}
uint32_t max_one_time_bonus(const frz_scoring& s) {  // src/lib.rs:497-503
    uint32_t bonus = std::max(s.delimiter_bonus, s.capitalization_bonus);
    uint32_t amort = std::max((bonus + 1) / 2, bonus > s.gap_open_penalty ? bonus - s.gap_open_penalty : 0u);
    return bonus - amort;
}
bool score_fits_in_u8(size_t needle_len, const frz_scoring& s) {  // src/smith_waterman/mod.rs:91-116
    size_t mc = (size_t)s.match_score + s.mismatch_penalty;
    mc = std::max<size_t>(mc, s.gap_open_penalty);
    mc = std::max<size_t>(mc, s.gap_extend_penalty);
    mc = std::max<size_t>(mc, s.matching_case_bonus);
    mc = std::max<size_t>(mc, s.capitalization_bonus);
    mc = std::max<size_t>(mc, s.delimiter_bonus);
    mc = std::max<size_t>(mc, s.prefix_bonus);
    if (mc > 255) return false;
    if (64 * (size_t)s.gap_extend_penalty + s.gap_open_penalty > 255) return false;
    size_t per_char = (size_t)s.match_score + max_per_char_bonus(s);
    size_t max_matrix = per_char * needle_len + max_one_time_bonus(s) + s.prefix_bonus;
    return max_matrix + s.mismatch_penalty <= 255;
}
// Scoring::guard_against_score_overflow (src/lib.rs:506-537)
frz_status guard_against_score_overflow(const frz_scoring& s, size_t needle_len, uint32_t max_bonus_per_char, uint32_t one_time) {
    uint32_t per_char = sat_add16(s.match_score, max_bonus_per_char);
    if (per_char == 0) return FRZ_OK;
    uint32_t headroom = sat_sub16(sat_sub16(sat_sub16(sat_sub16(0xFFFF, s.prefix_bonus), s.exact_match_bonus), s.mismatch_penalty), one_time);
    uint32_t max_len = headroom / per_char;
    if (needle_len > max_len)
        return frz_fail(FRZ_ERR_NEEDLE_TOO_LONG, "needle too long and could overflow the u16 score: %zu > %u", needle_len, max_len);
    size_t max_gap = 32 * (size_t)s.gap_extend_penalty + s.gap_open_penalty;
    if (max_gap > 0xFFFF)
        return frz_fail(FRZ_ERR_GAP_OVERFLOW, "gap penalties too large and could overflow the u16 score: %zu > 65535", max_gap);
    return FRZ_OK;
}

// case_needle (src/prefilter/mod.rs:49-65): the byte a needle byte also matches, an ASCII letter in the other case unless
// the match respects case
uint8_t case_flip(uint8_t ch, bool case_sensitive) {
    if (case_sensitive) return ch;
    if (ch >= 'a' && ch <= 'z') return (uint8_t)(ch - 32);
    if (ch >= 'A' && ch <= 'Z') return (uint8_t)(ch + 32);
    return ch;
}

// The byte classes (frz_device.cuh: frz_sig_bucket) that hold one / two or more of the needle's bytes.  On the unicode
// path only the needle's ASCII scalars count: a non-ASCII scalar and its case flip may differ in every byte, an ASCII
// scalar is matched by the same letter in either case, which the classes fold.
void sig_need_masks(const uint8_t* nd, size_t n, bool needs_unicode, FrzPatternDev* d) {
    uint32_t cnt[32] = {0};
    for (size_t i = 0; i < n; i++)
        if (!needs_unicode || nd[i] < 0x80) cnt[frz_sig_bucket(nd[i])]++;
    d->sig_need1 = d->sig_need2 = 0;
    for (int b = 0; b < 32; b++) {
        if (cnt[b] >= 1) d->sig_need1 |= 1u << b;
        if (cnt[b] >= 2) d->sig_need2 |= 1u << b;
    }
}

struct Compiled {
    FrzPatternDev dev;
    bool negated = false;
    bool literal = false;
    bool unicode = false;      // UNICODE = true specialisations (unicode.cu)
    FrzUNeedle un;             // case_needle_unicode (valid when `unicode`)
    FrzUScoring usc;
    uint32_t score_bound = 0;  // host-side upper bound of any score this pattern can emit
    // needle of more than FRZ_MAX_NEEDLE bytes: its per-position data (host copy), uploaded per device by pattern_for_launch
    std::shared_ptr<const FrzNeedleTab> tab;
    bool is_long() const { return dev.n > FRZ_MAX_NEEDLE; }
};

// Matcher::compile + get_backend (src/matcher/mod.rs:193-205, 448-498) → device pattern
frz_status compile_pattern(const OwnedPattern& src, const frz_config& mcfg, bool* is_none, Compiled* out) {
    *is_none = src.needle.empty();
    if (*is_none) return FRZ_OK;
    // PatternConfig::resolve (src/pattern.rs:250-262)
    const int max_typos = src.max_typos >= 0 ? src.max_typos : mcfg.max_typos;
    const int casing = src.casing >= 0 ? src.casing : mcfg.casing;
    const int unicode = src.unicode >= 0 ? src.unicode : mcfg.unicode;
    const int matching = src.matching >= 0 ? src.matching : mcfg.matching;
    const frz_scoring sc = src.has_scoring ? src.scoring : mcfg.scoring;
    const uint8_t* nd = (const uint8_t*)src.needle.data();
    const size_t n = src.needle.size();
    bool ascii = true;
    size_t nchars = 0;
    for (size_t i = 0; i < n; i++) {
        if (nd[i] >= 0x80) ascii = false;
        if ((nd[i] & 0xC0) != 0x80) nchars++;
    }
    // UnicodeMatching::respects_unicode_for (src/lib.rs:394-401)
    const bool needs_unicode = unicode == FRZ_UNICODE_ALWAYS || (unicode == FRZ_UNICODE_SMART && !ascii);
    // CaseMatching::respects_case_for (src/lib.rs:368-377): needle.chars().any(char::is_uppercase)
    bool case_sensitive;
    if (casing == FRZ_CASE_IGNORE) case_sensitive = false;
    else if (casing == FRZ_CASE_RESPECT) case_sensitive = true;
    else case_sensitive = frz_needle_has_uppercase(nd, n);
    if (n > FRZ_LONG_NEEDLE) return frz_fail(FRZ_ERR_UNSUPPORTED, "needle of %zu bytes exceeds the GPU kernels' limit of %d", n, FRZ_LONG_NEEDLE);
    if (n > FRZ_MAX_NEEDLE && needs_unicode)
        return frz_fail(FRZ_ERR_UNSUPPORTED, "needle of %zu bytes takes the unicode path, whose kernels handle up to %d bytes", n,
                        FRZ_MAX_NEEDLE);

    Compiled c;
    FrzPatternDev& d = c.dev;
    memset(&d, 0, sizeof d);
    c.negated = src.negated;
    c.literal = matching != FRZ_MATCHING_FUZZY;
    c.unicode = needs_unicode;
    if (needs_unicode) {
        if (!frz_build_uneedle(nd, n, case_sensitive, &c.un)) return frz_fail(FRZ_ERR_INVALID_ARG, "the needle is not valid UTF-8");
    } else {
        // byte path: only the byte-level case_needle pairs are used (frz_match_indices, which refuses long needles); the
        // needle may be any bytes
        memset(&c.un, 0, sizeof c.un);
        c.un.nbytes = (int32_t)n;
        for (size_t i = 0; i < n && i < FRZ_MAX_NEEDLE; i++) {
            const uint8_t ch = nd[i];
            c.un.c[i] = ch;
            c.un.f[i] = ch;
            c.un.bflip[i] = case_flip(ch, case_sensitive);
        }
    }
    d.n = (int)n;
    d.matching = matching;
    d.case_sensitive = case_sensitive;
    FrzNeedleTab tab;   // per-position data; FrzPatternDev keeps its first FRZ_MAX_NEEDLE positions
    memset(&tab, 0, sizeof tab);
    for (size_t i = 0; i < n; i++) {
        const uint8_t ch = nd[i], fl = case_flip(ch, case_sensitive);
        tab.c[i] = ch; tab.flip[i] = fl;
        tab.om[i] = fl != ch ? 0x20 : 0;
        tab.tg[i] = fl != ch ? (uint8_t)(ch | 0x20) : ch;
    }
    const size_t n_short = std::min<size_t>(n, FRZ_MAX_NEEDLE);
    memcpy(d.c, tab.c, n_short); memcpy(d.flip, tab.flip, n_short); memcpy(d.om, tab.om, n_short); memcpy(d.tg, tab.tg, n_short);
    if (n > FRZ_MAX_NEEDLE) c.tab = std::make_shared<const FrzNeedleTab>(tab);
    // distinct (om, tg) classes for the occurrence-mask prefilter.  A long needle takes the scanning forms (n_distinct 0):
    // over 64 bytes of ordinary text seldom stay within 16 classes.
    if (n <= FRZ_MAX_NEEDLE) {
        int nd = 0;
        bool ok = true;
        for (size_t i = 0; i < n && ok; i++) {
            int found = -1;
            for (int k = 0; k < nd; k++) if (d.dc_om[k] == d.om[i] && d.dc_tg[k] == d.tg[i]) { found = k; break; }
            if (found < 0) {
                if (nd == 16) { ok = false; break; }
                d.dc_om[nd] = d.om[i]; d.dc_tg[nd] = d.tg[i]; found = nd++;
            }
            d.cid[i] = (uint8_t)found;
        }
        d.n_distinct = ok ? nd : 0;
    }
    d.raw_match = sc.match_score; d.raw_mismatch = sc.mismatch_penalty; d.raw_gap_open = sc.gap_open_penalty;
    d.raw_gap_extend = sc.gap_extend_penalty; d.raw_prefix = sc.prefix_bonus; d.raw_cap = sc.capitalization_bonus;
    d.raw_case = sc.matching_case_bonus; d.raw_delim = sc.delimiter_bonus; d.exact_bonus = sc.exact_match_bonus;

    const CpuIsa isa = detect_isa();
    const int em = mcfg.emulate_lanes;
    if (em != 0 && em != 16 && em != 32 && em != 64) return frz_fail(FRZ_ERR_INVALID_ARG, "emulate_lanes must be 0, 16, 32 or 64");
    // per-char bound used for the sort's digit width
    const uint32_t maxb = std::max(sc.capitalization_bonus, sc.delimiter_bonus);

    memset(&c.usc, 0, sizeof c.usc);   // untruncated u16 scoring (literal matcher, greedy scorer); lane constants below
    c.usc.raw_match = sc.match_score; c.usc.raw_gap_open = sc.gap_open_penalty; c.usc.raw_gap_extend = sc.gap_extend_penalty;
    c.usc.raw_prefix = sc.prefix_bonus; c.usc.raw_cap = sc.capitalization_bonus; c.usc.raw_case = sc.matching_case_bonus;
    c.usc.raw_delim = sc.delimiter_bonus; c.usc.exact_bonus = sc.exact_match_bonus;
    if (c.literal) {
        // LiteralImpl::guard_against_score_overflow (src/literal/algo.rs:316-324)
        FRZ_TRY(guard_against_score_overflow(sc, n, sat_add16(maxb, sc.matching_case_bonus), 0));
        d.typo_mode = FRZ_T_LITERAL;
        d.min_hay_len = 0;
        // a literal match holds every needle byte (either case): signature test with no typo budget
        sig_need_masks(nd, n, needs_unicode, &d);
        d.sig_on = 1;
        d.sig_k = 0;
        d.pf_lanes = 64; d.sw_lanes = 64; d.score_bits = 16;
        uint64_t b = (uint64_t)n * ((uint64_t)sc.match_score + sc.matching_case_bonus + maxb) + sc.prefix_bonus + sc.exact_match_bonus;
        c.score_bound = (uint32_t)std::min<uint64_t>(b, 0xFFFF);
        *out = c;
        return FRZ_OK;
    }
    // MatcherImpl::guard_against_score_overflow (src/matcher/algo.rs:311-325): byte length on the ascii path,
    // (needle.chars().count() when the unicode specialisation is selected, algo.rs:318-321)
    const size_t guard_len = needs_unicode ? nchars : n;
    FRZ_TRY(guard_against_score_overflow(sc, guard_len, max_per_char_bonus(sc), max_one_time_bonus(sc)));
    const bool use_u8 = score_fits_in_u8(n, sc);
    int pf_lanes, sw_lanes;
    if (em == 0) {
        if (use_u8) {
            if (isa.avx512_pf && isa.avx512_sw_u8) { pf_lanes = 64; sw_lanes = 64; }
            else if (isa.avx2) { pf_lanes = 32; sw_lanes = 32; }
            else { pf_lanes = 16; sw_lanes = 16; }   // SSE / NEON / scalar
        } else {
            if (isa.avx512_pf && isa.avx512_sw) { pf_lanes = 64; sw_lanes = 32; }
            else if (isa.avx2) { pf_lanes = 32; sw_lanes = 16; }
            else { pf_lanes = 16; sw_lanes = 8; }
        }
    } else {
        pf_lanes = em;
        sw_lanes = use_u8 ? em : em / 2;
    }
    d.pf_lanes = pf_lanes; d.sw_lanes = sw_lanes; d.score_bits = use_u8 ? 8 : 16;
    // constants exactly as the reference splats them (ascii.rs:35-46); `as u8` truncation in the u8 family
    const uint32_t tm = use_u8 ? 0xFF : 0xFFFF;
    d.gap_extend = sc.gap_extend_penalty & tm;
    d.gap_open_x = sat_sub16(sc.gap_open_penalty, sc.gap_extend_penalty) & tm;
    d.match_x = sat_add16(sc.match_score, sc.mismatch_penalty) & tm;
    d.mismatch = sc.mismatch_penalty & tm;
    d.case_bonus = sc.matching_case_bonus & tm;
    d.cap_bonus = sc.capitalization_bonus & tm;
    d.delim_bonus = sc.delimiter_bonus & tm;
    d.prefix_bonus = sc.prefix_bonus & tm;
    c.usc.gex = d.gap_extend; c.usc.gopx = d.gap_open_x; c.usc.match_x = d.match_x; c.usc.mismatch = d.mismatch;
    c.usc.case_bonus = d.case_bonus; c.usc.cap_bonus = d.cap_bonus; c.usc.delim_bonus = d.delim_bonus; c.usc.prefix_bonus = d.prefix_bonus;
    {
        auto sp = [](int v) { return ((uint32_t)v & 0xffffu) * 0x00010001u; };
        for (int k = 0; k < 6; k++) {
            const int sft = 1 << k;
            d.k_pen_a[k] = sp(-(sft * d.gap_extend));
            d.k_pen_b[k] = sp(-(sft * d.gap_extend + d.gap_open_x));
        }
        d.k_neg_mis = sp(-d.mismatch);
        d.k_ex_add = sp(d.case_bonus - d.mismatch);
        d.k_up_plain = sp(-d.gap_extend);
        d.k_up_open = sp(-(d.gap_extend + d.gap_open_x));
        d.k_case = sp(d.case_bonus); d.k_cap = sp(d.cap_bonus); d.k_delim = sp(d.delim_bonus); d.k_base = sp(d.match_x);
        for (size_t i = 0; i < n_short; i++) { d.om16[i] = sp(d.om[i]); d.tg16[i] = sp(d.tg[i]); d.c16[i] = sp(d.c[i]); }
    }
    // the kernels keep cells in signed 16-bit lanes: every intermediate must stay below 2^15
    const uint64_t cell_bound = (uint64_t)n * ((uint64_t)sc.match_score + maxb + sc.matching_case_bonus) + sc.prefix_bonus +
                                (uint64_t)sc.mismatch_penalty + sc.match_score;
    const uint64_t pen_bound = (uint64_t)sw_lanes * sc.gap_extend_penalty + sc.gap_open_penalty;
    if (!needs_unicode && (cell_bound > 32767 || pen_bound > 32767))   // (the unicode kernel uses true u8/u16 lanes)
        return frz_fail(FRZ_ERR_UNSUPPORTED, "scoring/needle combination exceeds the kernels' signed 16-bit cell range");
    d.wrap8 = use_u8 && cell_bound > 255;  // cannot prove "no u8 add ever wraps" → emulate the wrap
    {   // column-limited SW classes need: padding bytes (0) never match, and plain (non-wrapping) arithmetic
        bool has_nul = false;
        for (size_t i = 0; i < n; i++) has_nul = has_nul || nd[i] == 0;
        d.col_classes = (!d.wrap8 && !has_nul) ? 1 : 0;
    }
    if (max_typos < 0) d.typo_mode = FRZ_T_NONE;
    else if (max_typos == 0) d.typo_mode = FRZ_T_0;
    else if (max_typos == 1) d.typo_mode = FRZ_T_1;
    else if (max_typos == 2) d.typo_mode = FRZ_T_2;
    else {
        d.typo_mode = FRZ_T_MANY;
        if (max_typos > 15 && (size_t)max_typos < guard_len)
            return frz_fail(FRZ_ERR_UNSUPPORTED, "max_typos > 15 is not on the GPU path yet");
    }
    {   // Phase-A necessary condition on the signature index (frz_device.cuh: frz_sig_bucket).  A haystack accepted with
        // k typos holds a common subsequence of n - k needle bytes (the k >= 1 trackers never accept what LCS rejects,
        // DESIGN.md §2), so per byte class at most k needle bytes in total may lack a partner:
        //     sum_c max(0, m_c - cnt_c) <= k     >=     popc(need1 & ~occurs) + popc(need2 & ~occurs_twice)
        // The unicode trackers are the same trackers over needle SCALARS; there only the ASCII scalars are counted
        // (sig_need_masks), which keeps the sum a lower bound.
        sig_need_masks(nd, n, needs_unicode, &d);
        d.sig_on = max_typos >= 0 ? 1 : 0;                       // NO_PREFILTER scores everything
        d.sig_k = max_typos < 0 ? 0 : std::min<int>(max_typos, 64);
    }
    d.max_typos = max_typos < 0 ? 0 : std::min(max_typos, (int)guard_len);  // budget >= needle length matches everything
    // min_haystack_len (src/matcher/algo.rs:62-65)
    d.min_hay_len = max_typos >= 0 ? (int)(nchars > (size_t)max_typos ? nchars - max_typos : 0) : 0;
    uint64_t b = std::min<uint64_t>(cell_bound, use_u8 ? 255 : 0xFFFF) + sc.exact_match_bonus;
    c.score_bound = (uint32_t)std::min<uint64_t>(b, 0xFFFF);
    *out = c;
    return FRZ_OK;
}

}  // namespace

struct frz_matcher {
    frz_config config;
    std::vector<OwnedPattern> raw;
    std::vector<Compiled> compiled;   // build_patterns: patterns with non-empty needles
    FrzWorkspace ws;
    // end-to-end (host in / host out) staging arena, grow-only: raw Arrow buffers + a reusable packed corpus
    FrzIngest e2e_ingest;     // staging arena + copy stream of frz_match_list_host*
    frz_corpus e2e_corpus;
    float last_ms[4] = {0, 0, 0, 0};
    uint64_t last_launches = 0;
    // shard path: the match count is known after the tile scan, long before the scores; it is published there so
    // that the count exchange of match_list_parallel overlaps the Smith-Waterman and sort kernels
    uint64_t* early_count_dst = nullptr;   // device destination of the count (set for the duration of a shard call)
    FrzEvent count_ev;                     // recorded once the count is in early_count_dst
    bool count_published = false;
    bool timings_pending = false;
    uint64_t epoch = 0;                    // identity of the compiled patterns (clones made for another epoch are stale)
    int last_sort_bins = 0;                // bins of the single-pass score sort of the last call (0: none / two passes)
    // the long needles' FrzNeedleTab, in pattern order, for the patterns of ntab_epoch
    FrzDevArray<FrzNeedleTab> ntab;
    uint64_t ntab_epoch = 0;
};

namespace {

std::atomic<uint64_t> g_matcher_epoch{1};

frz_status build_patterns(frz_matcher* m) {
    m->epoch = g_matcher_epoch.fetch_add(1);
    std::vector<Compiled> comp;
    for (const auto& p : m->raw) {
        bool none = false;
        Compiled c;
        FRZ_TRY(compile_pattern(p, m->config, &none, &c));
        if (!none) comp.push_back(c);
    }
    m->compiled.swap(comp);
    return FRZ_OK;
}

frz_status validate_config(const frz_config* c) {
    if (!c) return frz_fail(FRZ_ERR_INVALID_ARG, "null config");
    if (c->max_typos < -1 || c->max_typos > 65535) return frz_fail(FRZ_ERR_INVALID_ARG, "max_typos out of range");
    if (c->casing > 2 || c->unicode > 2 || c->matching > 4 || c->sort > 3) return frz_fail(FRZ_ERR_INVALID_ARG, "bad enum value in config");
    return FRZ_OK;
}

}  // namespace

extern "C" frz_status frz_matcher_create(const frz_pattern* patterns, size_t n_patterns, const frz_config* config, frz_matcher** out) {
    if (!out || (n_patterns && !patterns)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(validate_config(config));
    for (size_t i = 0; i < n_patterns; i++) {   // PatternConfig overrides (src/pattern.rs:230-246): -1 = inherit, else the enum range
        const frz_pattern& p = patterns[i];
        if (p.needle_len && !p.needle) return frz_fail(FRZ_ERR_INVALID_ARG, "pattern %zu: null needle", i);
        if (p.casing < -1 || p.casing > 2 || p.unicode < -1 || p.unicode > 2 || p.matching < -1 || p.matching > 4)
            return frz_fail(FRZ_ERR_INVALID_ARG, "pattern %zu: bad enum value in the per-pattern overrides", i);
        if (p.max_typos < -1 || p.max_typos > 65535) return frz_fail(FRZ_ERR_INVALID_ARG, "pattern %zu: max_typos out of range", i);
    }
    auto m = std::make_unique<frz_matcher>();
    m->config = *config;
    for (size_t i = 0; i < n_patterns; i++) {
        const frz_pattern& p = patterns[i];
        OwnedPattern o;
        o.needle.assign((const char*)p.needle, p.needle_len);
        o.raw = o.needle;
        o.negated = p.negated != 0;
        o.matching = p.matching; o.casing = p.casing; o.unicode = p.unicode; o.max_typos = p.max_typos;
        o.has_scoring = p.has_scoring != 0; o.scoring = p.scoring;
        m->raw.push_back(std::move(o));
    }
    FRZ_TRY(build_patterns(m.get()));
    *out = m.release();
    return FRZ_OK;
}

extern "C" frz_status frz_matcher_from_query(const uint8_t* query, size_t len, const frz_config* config, frz_matcher** out) {
    if (!out || (!query && len)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(validate_config(config));
    auto m = std::make_unique<frz_matcher>();
    m->config = *config;
    m->raw = parse_query(query, len);
    FRZ_TRY(build_patterns(m.get()));
    *out = m.release();
    return FRZ_OK;
}

extern "C" frz_status frz_matcher_set_config(frz_matcher* m, const frz_config* config) {
    if (!m) return frz_fail(FRZ_ERR_INVALID_ARG, "null matcher");
    FRZ_TRY(validate_config(config));
    if (memcmp(&m->config, config, sizeof *config) == 0) return FRZ_OK;
    frz_config old = m->config;
    m->config = *config;
    frz_status s = build_patterns(m);
    if (s != FRZ_OK) { m->config = old; build_patterns(m); }
    return s;
}

// `Matcher: Clone` (src/matcher/mod.rs:76): same patterns and config, fresh device scratch.  match_list_parallel clones
// the matcher once per worker (src/matcher/parallel.rs:46); frz_match_list_parallel does the same once per GPU.
extern "C" frz_status frz_matcher_clone(const frz_matcher* src, frz_matcher** out) {
    if (!src || !out) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    auto m = std::make_unique<frz_matcher>();
    m->config = src->config;
    m->raw = src->raw;
    FRZ_TRY(build_patterns(m.get()));
    *out = m.release();
    return FRZ_OK;
}
uint64_t frz_matcher_epoch(const frz_matcher* m) { return m ? m->epoch : 0; }
uint8_t frz_matcher_sort(const frz_matcher* m) { return m ? m->config.sort : 0; }
cudaEvent_t frz_matcher_table_event(const frz_matcher* m) {
    return (m && m->last_sort_bins && m->ws.sort.table_ev_recorded) ? m->ws.sort.table_ev.get() : nullptr;
}
const uint32_t* frz_matcher_last_sort_table(const frz_matcher* m, int* bins) {
    if (bins) *bins = m ? m->last_sort_bins : 0;
    return (m && m->last_sort_bins) ? frz_sort_digit_base(m->ws.sort) : nullptr;
}

extern "C" void frz_matcher_destroy(frz_matcher* m) { delete m; }
extern "C" size_t frz_matcher_num_patterns(const frz_matcher* m) { return m ? m->compiled.size() : 0; }
extern "C" frz_status frz_matcher_backend_info(const frz_matcher* m, size_t i, int* lanes, int* score_bits, int* prefilter_lanes, int* is_literal) {
    if (!m || i >= m->compiled.size()) return frz_fail(FRZ_ERR_INVALID_ARG, "pattern index out of range");
    const auto& c = m->compiled[i];
    if (lanes) *lanes = c.dev.sw_lanes;
    if (score_bits) *score_bits = c.dev.score_bits;
    if (prefilter_lanes) *prefilter_lanes = c.dev.pf_lanes;
    if (is_literal) *is_literal = c.literal;
    return FRZ_OK;
}
void collect_timings(frz_matcher* m, const FrzLaunchStats& st);
extern "C" frz_status frz_matcher_last_timings(const frz_matcher* mc, float* ms4, uint64_t* launches) {
    frz_matcher* m = const_cast<frz_matcher*>(mc);
    if (!m) return frz_fail(FRZ_ERR_INVALID_ARG, "null matcher");
    if (m->timings_pending && m->ws.device >= 0) {
        cudaSetDevice(m->ws.device);
        cudaEventSynchronize(m->ws.ev[3].get());
        FrzLaunchStats st;
        st.launches = m->last_launches;
        collect_timings(m, st);
        m->timings_pending = false;
    }
    if (ms4) memcpy(ms4, m->last_ms, sizeof m->last_ms);
    if (launches) *launches = m->last_launches;
    return FRZ_OK;
}

// ------------------------------------------------------------------------ small helper kernels

namespace {

__global__ void k_fill_all(FrzMatchDev* out, uint64_t n, uint32_t index_offset, FrzCounters* ctr) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        out[i] = FrzMatchDev{index_offset + (uint32_t)i, 0, 0, 0};
    if (blockIdx.x == 0 && threadIdx.x == 0) ctr->total = n;
}
__global__ void k_reverse(const FrzMatchDev* in, FrzMatchDev* out, const unsigned long long* n_ptr) {
    const unsigned long long n = *n_ptr;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        out[n - 1 - i] = in[i];
}
// keep[i] = candidate i is (not) hit; hits are index-ordered → binary search
__device__ __forceinline__ long long find_hit(const FrzMatchDev* hits, uint64_t nh, uint32_t index) {
    uint64_t lo = 0, hi = nh;
    while (lo < hi) {
        uint64_t mid = (lo + hi) >> 1;
        if (hits[mid].index < index) lo = mid + 1; else hi = mid;
    }
    return (lo < nh && hits[lo].index == index) ? (long long)lo : -1;
}
// non-negated extra pattern: every hit is a surviving candidate; add the candidate's score
// (hit.score saturating_add, exact |=; src/matcher/multi.rs:133-147)
__global__ void k_combine_hits(const FrzMatchDev* cand, uint64_t nc, FrzMatchDev* hits, uint64_t nh) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nh; i += (uint64_t)gridDim.x * blockDim.x) {
        FrzMatchDev h = hits[i];
        long long j = find_hit(cand, nc, h.index);
        if (j >= 0) {
            uint32_t s = (uint32_t)h.score + cand[j].score;
            h.score = (uint16_t)(s > 0xFFFF ? 0xFFFF : s);
            h.exact |= cand[j].exact;
        }
        hits[i] = h;
    }
}
// haystack idx's slot is in use: it was not removed (frz_corpus_remove), and a subset call's masked metadata keeps it
__device__ __forceinline__ bool slot_in_use(const uint32_t* __restrict__ slot_meta, const uint16_t* __restrict__ slot_of, uint64_t idx) {
    return slot_meta[(idx & ~(uint64_t)(FRZ_TILE - 1)) + slot_of[idx]] != FRZ_INVALID_SLOT;
}

// Stable compaction of a list: per-block ballot counts (k_keep) → single-block scan → scatter.  The row rules of k_keep:
// negated extra pattern: retain the candidates that were NOT hit (src/matcher/multi.rs:124-132)
struct NotHit {
    const FrzMatchDev* cand;
    const FrzMatchDev* hits;
    uint64_t nh;
    __device__ bool operator()(uint64_t i) const { return find_hit(hits, nh, cand[i].index) < 0; }
};
// a k_fill_all list (row i = haystack i): retain the haystacks whose slot is in use
struct LiveIndex {
    const uint32_t* slot_meta;
    const uint16_t* slot_of;
    __device__ bool operator()(uint64_t i) const { return slot_in_use(slot_meta, slot_of, i); }
};
// the list form of a subset call: cand[i] = member i as a match record, retained when its slot is in use (removed members
// are dropped: the candidate-list prefilter reads their slot metadata unchecked)
struct LiveMember {
    const uint32_t* members;
    const uint32_t* slot_meta;
    const uint16_t* slot_of;
    FrzMatchDev* cand;
    __device__ bool operator()(uint64_t i) const {
        const uint32_t idx = members[i];
        cand[i] = FrzMatchDev{idx, 0, 0, 0};
        return slot_in_use(slot_meta, slot_of, idx);
    }
};
constexpr int kCompactBlock = 1024;
// keep[i] = rule(i) for the n rows, and the kept rows of each block → block_count
template <class Rule>
__global__ void __launch_bounds__(kCompactBlock) k_keep(Rule rule, uint64_t n, uint32_t* block_count, uint8_t* keep) {
    __shared__ uint32_t wc[32];
    const uint64_t i = (uint64_t)blockIdx.x * kCompactBlock + threadIdx.x;
    const bool k = i < n && rule(i);
    if (i < n) keep[i] = k;
    const uint32_t b = __ballot_sync(0xffffffffu, k);
    if ((threadIdx.x & 31) == 0) wc[threadIdx.x >> 5] = __popc(b);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int w = 0; w < 32; w++) s += wc[w];
        block_count[blockIdx.x] = s;
    }
}
__global__ void __launch_bounds__(kCompactBlock) k_retain_scatter(const FrzMatchDev* cand, uint64_t nc, const uint8_t* keep,
                                                                  const uint64_t* block_base, FrzMatchDev* out) {
    __shared__ uint32_t wc[32];
    uint64_t i = (uint64_t)blockIdx.x * kCompactBlock + threadIdx.x;
    bool k = i < nc && keep[i];
    uint32_t b = __ballot_sync(0xffffffffu, k);
    uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) wc[warp] = __popc(b);
    __syncthreads();
    uint32_t pre = 0;
    for (uint32_t w = 0; w < warp; w++) pre += wc[w];
    if (k) out[block_base[blockIdx.x] + pre + __popc(b & ((1u << lane) - 1))] = cand[i];
}
__global__ void __launch_bounds__(1024) k_scan_blocks(const uint32_t* cnt, uint64_t* base, uint32_t n, FrzCounters* ctr) {
    __shared__ uint64_t carry;
    __shared__ uint64_t ws[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t b0 = 0; b0 < n; b0 += blockDim.x) {
        uint32_t i = b0 + threadIdx.x;
        uint64_t v = i < n ? cnt[i] : 0, x = v;
        for (int d = 1; d < 32; d <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, x, d); if ((threadIdx.x & 31) >= (unsigned)d) x += y; }
        if ((threadIdx.x & 31) == 31) ws[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint64_t w = ws[threadIdx.x], xs = w;
            for (int d = 1; d < 32; d <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, xs, d); if (threadIdx.x >= (unsigned)d) xs += y; }
            ws[threadIdx.x] = xs - w;
        }
        __syncthreads();
        uint64_t incl = carry + ws[threadIdx.x >> 5] + x;
        if (i < n) base[i] = incl - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) ctr->total = carry;
}
// Slot metadata of a subset call: slot s keeps its metadata when its haystack, index (s & ~1023) + (meta & 1023), is below
// n_bits with its bit set in `bits`; every other slot becomes FRZ_INVALID_SLOT, which the matching kernels skip.  Four
// slots of one tile per thread (n_slots is a multiple of FRZ_TILE).
__global__ void k_subset_meta(const uint4* __restrict__ slot_meta, uint64_t n_quads, const uint32_t* __restrict__ bits, uint64_t n_bits,
                              uint4* __restrict__ out) {
    for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n_quads; q += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t tile0 = (q * 4) & ~(uint64_t)(FRZ_TILE - 1);
        uint32_t v[4];
        *reinterpret_cast<uint4*>(v) = slot_meta[q];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint64_t idx = tile0 + (v[j] & (FRZ_TILE - 1));
            if (v[j] == FRZ_INVALID_SLOT || idx >= n_bits || !((bits[idx >> 5] >> (idx & 31)) & 1u)) v[j] = FRZ_INVALID_SLOT;
        }
        out[q] = *reinterpret_cast<const uint4*>(v);
    }
}

frz_status ensure_workspace(frz_matcher* m, const FrzCorpusStorage& cs, uint64_t survivor_cap) {
    FrzWorkspace& ws = m->ws;
    if (ws.device != cs.device) {   // all or nothing: a failed set-up leaves an empty workspace, redone by the next call
        ws = FrzWorkspace();         // the old device's buffers go first
        FRZ_CUDA_TRY(cudaSetDevice(cs.device));
        FrzWorkspace fresh;
        fresh.device = cs.device;
        FRZ_TRY(fresh.counters.reserve(1));
        FRZ_TRY(fresh.stream_total.reserve(2));
        FRZ_TRY(fresh.h_counters.reserve(1));
        for (auto& e : fresh.ev) FRZ_TRY(frz_event_create(e, cudaEventDefault));
        FRZ_TRY(frz_event_create(fresh.sort.table_ev, cudaEventDisableTiming));
        FRZ_TRY(frz_sort_hist_alloc(fresh.sort.hist));
        ws = std::move(fresh);
    }
    FRZ_TRY(ws.surv_bitmap.reserve((size_t)cs.n_tiles * 32));
    FRZ_TRY(ws.word_prefix.reserve((size_t)cs.n_tiles * 32));
    FRZ_TRY(ws.tile_count.reserve(cs.n_tiles));
    FRZ_TRY(ws.tile_out_base.reserve(cs.n_tiles));
    for (auto& s : ws.survivors) FRZ_TRY(s.reserve(survivor_cap));
    FRZ_TRY(ws.cand_list.reserve(std::max<uint64_t>(cs.n, 1)));   // worst case: every haystack passes the signature test
    FRZ_TRY(ws.matches_a.reserve(cs.n, std::max<uint64_t>(cs.n, 1)));
    FRZ_TRY(ws.matches_b.reserve(cs.n, std::max<uint64_t>(cs.n, 1)));
    return FRZ_OK;
}

// multi-pattern candidate ping-pong / two-pass sort scratch: grow-only, always >= n entries after this call
frz_status ensure_multi_buffers(frz_matcher* m, uint64_t n) {
    FRZ_TRY(m->ws.multi_a.reserve(std::max<uint64_t>(n, 1)));
    return m->ws.multi_b.reserve(std::max<uint64_t>(n, 1));
}

// stable-compaction scratch (k_keep → k_scan_blocks → k_retain_scatter) for lists of up to n entries
frz_status ensure_retain_buffers(frz_matcher* m, uint64_t n) {
    FrzWorkspace& ws = m->ws;
    if (ws.retain_keep.cap() >= n) return FRZ_OK;
    const uint32_t nb_max = (uint32_t)((n + kCompactBlock - 1) / kCompactBlock) + 1;
    FRZ_TRY(ws.retain_cnt.reserve(nb_max));
    FRZ_TRY(ws.retain_base.reserve(nb_max));
    return ws.retain_keep.reserve(n);
}

// Stable compaction of the n >= 1 rows of `in`: the rows that `rule` keeps → `out`, in order, their count →
// ws.counters->total.
template <class Rule>
frz_status retain_rows(frz_matcher* m, Rule rule, const FrzMatchDev* in, uint64_t n, FrzMatchDev* out, cudaStream_t stream,
                       FrzLaunchStats* st) {
    FrzWorkspace& ws = m->ws;
    FRZ_TRY(ensure_retain_buffers(m, n));
    const uint32_t nb = (uint32_t)((n + kCompactBlock - 1) / kCompactBlock);
    k_keep<<<nb, kCompactBlock, 0, stream>>>(rule, n, ws.retain_cnt.get(), ws.retain_keep.get());
    k_scan_blocks<<<1, 1024, 0, stream>>>(ws.retain_cnt.get(), ws.retain_base.get(), nb, ws.counters.get());
    k_retain_scatter<<<nb, kCompactBlock, 0, stream>>>(in, n, ws.retain_keep.get(), ws.retain_base.get(), out);
    st->launches += 3;
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

uint64_t initial_survivor_cap(const FrzCorpusStorage& cs, const FrzPatternDev& d) {
    if (d.typo_mode == FRZ_T_NONE) return std::max<uint64_t>(cs.n, 1);
    return std::min<uint64_t>(std::max<uint64_t>(cs.n / 4, 1 << 16), std::max<uint64_t>(cs.n, 1));
}

// A long needle's FrzNeedleTab on the workspace's device, uploaded once per compiled pattern set (build_patterns starts a
// new epoch) and device; nullptr for other needles.
frz_status needle_table(frz_matcher* m, const Compiled& c, const FrzNeedleTab** out) {
    *out = nullptr;
    if (!c.is_long()) return FRZ_OK;
    if (!m->ntab.get() || m->ntab.device() != m->ws.device || m->ntab_epoch != m->epoch) {
        m->ntab.reset();
        m->ntab_epoch = 0;
        size_t k = 0;
        for (const Compiled& p : m->compiled) k += p.is_long() ? 1 : 0;
        FRZ_TRY(m->ntab.reserve(k));
        k = 0;
        for (const Compiled& p : m->compiled)
            if (p.is_long()) FRZ_CUDA_TRY(cudaMemcpy(m->ntab.get() + k++, p.tab.get(), sizeof(FrzNeedleTab), cudaMemcpyHostToDevice));
        m->ntab_epoch = m->epoch;
    }
    size_t k = 0;
    for (const Compiled& p : m->compiled) {
        if (&p == &c) break;
        k += p.is_long() ? 1 : 0;
    }
    *out = m->ntab.get() + k;
    return FRZ_OK;
}

// timing event i of the current call (FrzWorkspace::ev)
void record_ev(FrzWorkspace& ws, int i, cudaStream_t stream) {
    cudaEventRecord(ws.ev[i].get(), stream);
    ws.ev_rec[i] = true;
}

// the start of a match call: no timing event recorded yet, no single-pass sort table
void reset_call_state(frz_matcher* m) {
    for (bool& f : m->ws.ev_rec) f = false;
    m->last_sort_bins = 0;
}

// shard calls: ws.counters->total → *dst, then count_ev
frz_status publish_count(frz_matcher* m, uint64_t* dst, cudaStream_t stream) {
    FRZ_CUDA_TRY(cudaMemcpyAsync(dst, &m->ws.counters.get()->total, sizeof(uint64_t), cudaMemcpyDeviceToDevice, stream));
    FRZ_CUDA_TRY(cudaEventRecord(m->count_ev.get(), stream));
    m->count_published = true;
    return FRZ_OK;
}

// An asynchronous shard call: body(&st) enqueues the call's work on `stream`.  Meanwhile the count goes to d_count as soon
// as it is known (the body publishes it early where it can, else it is published after the body) and the score sort
// records its table event.  frz_matcher_last_timings reads the events once the stream is idle.
template <class Body>
frz_status shard_call(frz_matcher* m, uint64_t* d_count, cudaStream_t stream, Body&& body) {
    if (!m->count_ev) FRZ_TRY(frz_event_create(m->count_ev, cudaEventDisableTiming));
    FrzLaunchStats st;
    m->early_count_dst = d_count;
    m->count_published = false;
    m->ws.sort.arm_table_ev = true;
    m->ws.sort.table_ev_recorded = false;
    const frz_status s = body(&st);
    m->early_count_dst = nullptr;
    m->ws.sort.arm_table_ev = false;
    FRZ_TRY(s);
    if (!m->count_published) FRZ_TRY(publish_count(m, d_count, stream));
    m->last_launches = st.launches;
    m->timings_pending = true;
    return FRZ_OK;
}

// One pattern over the corpus (optionally restricted to a candidate list) → index-ordered matches in d_out (reversed
// order if `reversed`); the count is left in ws.counters->total (device).  masked_meta (subset calls): slot metadata to
// read in place of the corpus's own, nullptr = the corpus's.
frz_status run_pattern(frz_matcher* m, const FrzCorpusStorage& cs, const Compiled& c, const uint32_t* masked_meta,
                       uint32_t index_offset, bool reversed, FrzMatchDev* d_out, cudaStream_t stream, FrzLaunchStats* st,
                       bool record_events, const FrzMatchDev* cand_list = nullptr, uint64_t n_cand = 0,
                       const FrzScoreHist& hist = FrzScoreHist()) {
    FrzWorkspace& ws = m->ws;
    FrzCorpusView cv = cs.view();
    if (masked_meta) cv.slot_meta = masked_meta;
    uint64_t cap = std::max(ws.survivor_cap(), initial_survivor_cap(cs, c.dev));
    FRZ_TRY(ensure_workspace(m, cs, cap));
    const FrzNeedleTab* ntab = nullptr;
    FRZ_TRY(needle_table(m, c, &ntab));
    FRZ_CUDA_TRY(cudaMemsetAsync(ws.counters.get(), 0, sizeof(FrzCounters), stream));
    if (record_events) record_ev(ws, 0, stream);
    if (c.unicode) FRZ_TRY(frz_launch_unicode(cv, c.dev, c.un, c.usc, cand_list, n_cand, index_offset, ws, stream, st));
    else if (cand_list) FRZ_TRY(frz_launch_prefilter_list(cv, c.dev, cand_list, n_cand, index_offset, ws, stream, st, ntab));
    else FRZ_TRY(frz_launch_prefilter(cv, c.dev, ws, stream, st, ntab));
    FRZ_TRY(frz_launch_tile_scan(cv, ws, stream, st));
    if (record_events) record_ev(ws, 1, stream);
    // single pattern: every survivor becomes exactly one match, so the scan total is the final count
    if (m->early_count_dst && !cand_list && m->compiled.size() == 1) FRZ_TRY(publish_count(m, m->early_count_dst, stream));
    // A survivor-list overflow (lists are sized by a heuristic unless the pattern can match everything)
    // only sets a sticky device flag; whoever reads the counters back re-runs with worst-case lists.
    if (c.unicode) {
        // the unicode kernel has already scored its survivors: they travel as literal-style records (score, exact)
        FrzPatternDev emit = c.dev;
        emit.typo_mode = FRZ_T_LITERAL;
        FRZ_TRY(frz_launch_sw(cv, emit, index_offset, reversed, ws, d_out, stream, st, hist));
    } else {
        FRZ_TRY(frz_launch_sw(cv, c.dev, index_offset, reversed, ws, d_out, stream, st, hist, ntab));
    }
    if (record_events) record_ev(ws, 2, stream);
    return FRZ_OK;
}

constexpr frz_status kRetryOverflow = (frz_status)100;

frz_status read_counters(frz_matcher* m, cudaStream_t stream) {
    FrzWorkspace& ws = m->ws;
    FRZ_CUDA_TRY(cudaMemcpyAsync(ws.h_counters.get(), ws.counters.get(), sizeof(FrzCounters), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    if (ws.h_counters.get()->error & FRZ_DEVERR_SURVIVOR_OVERFLOW) return kRetryOverflow;
    return FRZ_OK;
}

// Every index of the corpus, ascending, into `out` (count in ws.counters->total): the list of the empty matcher and the
// start of an all-negated one.  A corpus with removed haystacks, or a subset call (masked_meta, as in run_pattern), fills
// `tmp` and keeps only the indices whose slot is in use.
frz_status fill_all(frz_matcher* m, const FrzCorpusStorage& cs, uint32_t index_offset, FrzMatchDev* out, FrzMatchDev* tmp,
                    cudaStream_t stream, FrzLaunchStats* st, const uint32_t* masked_meta = nullptr) {
    FrzWorkspace& ws = m->ws;
    const bool filter = cs.n_removed || masked_meta;
    k_fill_all<<<grid_for(cs.n, 256), 256, 0, stream>>>(filter ? tmp : out, cs.n, index_offset, ws.counters.get());
    st->launches++;
    if (filter && cs.n)
        FRZ_TRY(retain_rows(m, LiveIndex{masked_meta ? masked_meta : cs.slot_meta.get(), cs.slot_of.get()}, tmp, cs.n, out, stream, st));
    FRZ_CUDA_TRY(cudaGetLastError());
    return FRZ_OK;
}

// The rows of a subset call, in one of two forms (DESIGN.md §4.9): slot metadata in which non-members are unused slots
// (masked form), or the live members, index-ordered, as a candidate list (list form).  The default scope is the whole
// corpus.  none: no row can match (the list form found no member in use), the call returns an empty list without running
// the pipeline.
struct SubsetScope {
    const uint32_t* masked_meta = nullptr;
    const FrzMatchDev* list = nullptr;
    uint64_t n_list = 0;
    bool none = false;
};

// a count known on the host → ws.counters->total
frz_status set_count(frz_matcher* m, uint64_t n, cudaStream_t stream) {
    FrzWorkspace& ws = m->ws;
    ws.h_counters.get()->total = n;
    FRZ_CUDA_TRY(cudaMemcpyAsync(&ws.counters.get()->total, &ws.h_counters.get()->total, sizeof(unsigned long long), cudaMemcpyHostToDevice, stream));
    return FRZ_OK;
}

// the list form's members → `out` as the start of a list, count → ws.counters->total
frz_status copy_scope_list(frz_matcher* m, const SubsetScope& scope, FrzMatchDev* out, cudaStream_t stream) {
    FRZ_CUDA_TRY(cudaMemcpyAsync(out, scope.list, scope.n_list * sizeof(FrzMatchDev), cudaMemcpyDeviceToDevice, stream));
    return set_count(m, scope.n_list, stream);
}

// match_list_into over all compiled patterns → index-ordered device list; returns pointer + leaves the
// count in ws.counters->total.  `final_reversed` asks for the list in descending index order.  `score_hist` (optional):
// the caller will sort the list by score; where the scoring kernels emit the list directly and one sort pass will do,
// they also build the sort's histogram, returned there (score_hist->counts stays nullptr otherwise).  scope: the rows of
// a subset call.  The list form's base pattern takes the members as its candidate list, and the empty and all-negated
// matchers start from them.
frz_status match_into_device(frz_matcher* m, const FrzCorpusStorage& cs, uint32_t index_offset, bool final_reversed,
                             FrzMatchDev** d_result, uint32_t* score_bound, cudaStream_t stream, FrzLaunchStats* st,
                             FrzMatchDev* prefer_out = nullptr, FrzScoreHist* score_hist = nullptr,
                             const SubsetScope& scope = SubsetScope()) {
    FrzWorkspace& ws = m->ws;
    const uint32_t* masked_meta = scope.masked_meta;
    FRZ_TRY(frz_check_index_range(cs.n, index_offset));
    const auto& pats = m->compiled;
    *score_bound = 0;
    if (pats.empty()) {  // CompiledPatterns::Empty (src/matcher/mod.rs:380-383)
        FRZ_TRY(ensure_workspace(m, cs, 1));
        FRZ_CUDA_TRY(cudaMemsetAsync(ws.counters.get(), 0, sizeof(FrzCounters), stream));
        if (scope.list) FRZ_TRY(copy_scope_list(m, scope, ws.matches_a.get(), stream));
        else FRZ_TRY(fill_all(m, cs, index_offset, ws.matches_a.get(), ws.matches_b.get(), stream, st, masked_meta));
        if (final_reversed) {
            k_reverse<<<grid_for(cs.n, 256), 256, 0, stream>>>(ws.matches_a.get(), ws.matches_b.get(), &ws.counters.get()->total);
            st->launches++;
            *d_result = ws.matches_b.get();
        } else *d_result = ws.matches_a.get();
        FRZ_CUDA_TRY(cudaGetLastError());
        return FRZ_OK;
    }
    if (pats.size() == 1 && !pats[0].negated) {  // CompiledPatterns::Single
        FRZ_TRY(ensure_workspace(m, cs, initial_survivor_cap(cs, pats[0].dev)));
        FrzMatchDev* dst = prefer_out ? prefer_out : ws.matches_a.get();
        FrzScoreHist hist;
        if (score_hist && frz_sort_single_pass_bins(pats[0].score_bound) > 0) {
            FRZ_TRY(frz_sort_fused_prepare(ws.sort, cs.n, pats[0].score_bound, stream, &hist));
            *score_hist = hist;
        }
        FRZ_TRY(run_pattern(m, cs, pats[0], masked_meta, index_offset, final_reversed, dst, stream, st, true, scope.list, scope.n_list,
                            hist));
        *d_result = dst;
        *score_bound = pats[0].score_bound;
        return FRZ_OK;
    }
    // CompiledPatterns::Multi (src/matcher/multi.rs:84-152).  Counts are read back between patterns.
    FRZ_TRY(ensure_workspace(m, cs, initial_survivor_cap(cs, pats[0].dev)));
    FRZ_TRY(ensure_multi_buffers(m, cs.n));
    int base = -1;
    for (size_t i = 0; i < pats.size(); i++) if (!pats[i].negated) { base = (int)i; break; }
    FrzMatchDev* cand = ws.multi_a.get();
    FrzMatchDev* spare = ws.multi_b.get();
    uint64_t nc = 0;
    uint64_t bound = 0;
    if (base >= 0) {
        FRZ_TRY(run_pattern(m, cs, pats[base], masked_meta, index_offset, false, cand, stream, st, true, scope.list, scope.n_list));
        FRZ_TRY(read_counters(m, stream));
        nc = ws.h_counters.get()->total;
        bound = pats[base].score_bound;
    } else if (scope.list) {
        FRZ_TRY(copy_scope_list(m, scope, cand, stream));
        nc = scope.n_list;
    } else {
        FRZ_CUDA_TRY(cudaMemsetAsync(ws.counters.get(), 0, sizeof(FrzCounters), stream));
        FRZ_TRY(fill_all(m, cs, index_offset, cand, spare, stream, st, masked_meta));
        if (masked_meta) {   // the members in use are counted on the device
            FRZ_TRY(read_counters(m, stream));
            nc = ws.h_counters.get()->total;
        } else nc = cs.n - cs.n_removed;
    }
    FRZ_TRY(ensure_retain_buffers(m, cs.n));   // once, for every negated pattern below
    frz_status status = FRZ_OK;
    for (size_t pi = 0; pi < pats.size() && status == FRZ_OK; pi++) {
        if ((int)pi == base || nc == 0) continue;
        status = [&]() -> frz_status {
            // evaluate the pattern on the surviving candidates only; hits land in ws.matches_a, index-ordered,
            // with real indices
            FRZ_TRY(run_pattern(m, cs, pats[pi], nullptr, index_offset, false, ws.matches_a.get(), stream, st, false, cand, nc));
            FRZ_TRY(read_counters(m, stream));
            const uint64_t nh = ws.h_counters.get()->total;
            if (pats[pi].negated) {
                FRZ_TRY(retain_rows(m, NotHit{cand, ws.matches_a.get(), nh}, cand, nc, spare, stream, st));
                FRZ_TRY(read_counters(m, stream));
                nc = ws.h_counters.get()->total;
                std::swap(cand, spare);
            } else {
                k_combine_hits<<<grid_for(nh, 256), 256, 0, stream>>>(cand, nc, ws.matches_a.get(), nh);
                st->launches++;
                FRZ_CUDA_TRY(cudaMemcpyAsync(spare, ws.matches_a.get(), nh * sizeof(FrzMatchDev), cudaMemcpyDeviceToDevice, stream));
                std::swap(cand, spare);
                nc = nh;
                bound += pats[pi].score_bound;
            }
            return FRZ_OK;
        }();
    }
    FRZ_TRY(status);
    // publish: count → counters.total, list → matches_a (reversed if asked)
    FRZ_TRY(set_count(m, nc, stream));
    if (final_reversed) {
        k_reverse<<<grid_for(nc, 256), 256, 0, stream>>>(cand, ws.matches_a.get(), &ws.counters.get()->total);
        st->launches++;
    } else {
        FRZ_CUDA_TRY(cudaMemcpyAsync(ws.matches_a.get(), cand, nc * sizeof(FrzMatchDev), cudaMemcpyDeviceToDevice, stream));
    }
    FRZ_CUDA_TRY(cudaGetLastError());
    *d_result = ws.matches_a.get();
    *score_bound = (uint32_t)std::min<uint64_t>(bound, 0xFFFF);
    return FRZ_OK;
}

// Matcher::match_list on device: into (+reverse) (+stable score sort).  Result pointer + device count.
__global__ void k_copy_n(const FrzMatchDev* __restrict__ in, FrzMatchDev* __restrict__ out, const unsigned long long* n_ptr,
                         uint32_t limit) {
    const unsigned long long n = min(*n_ptr, (unsigned long long)limit);
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        out[i] = in[i];
}

// `final_out` (optional, device, >= corpus length): where the final list must land.  `limit` (top-K calls): only the first
// `limit` positions of the final list are written (the sort's last scatter and the final copy drop the rest); the count in
// ws.counters->total stays the full match count.  scope: as in match_into_device.
frz_status match_list_device(frz_matcher* m, const FrzCorpusStorage& cs, uint32_t index_offset, uint8_t sort,
                             FrzMatchDev** d_result, cudaStream_t stream, FrzLaunchStats* st, FrzMatchDev* final_out = nullptr,
                             uint32_t limit = kFrzNoLimit, const SubsetScope& scope = SubsetScope()) {
    FrzWorkspace& ws = m->ws;
    const bool reversed = sort == FRZ_SORT_INDEX_DESC || sort == FRZ_SORT_SCORE_THEN_INDEX_DESC;
    const bool by_score = sort == FRZ_SORT_SCORE_THEN_INDEX_ASC || sort == FRZ_SORT_SCORE_THEN_INDEX_DESC;
    const bool will_sort = by_score && !m->compiled.empty();
    reset_call_state(m);
    FrzMatchDev* d_list = nullptr;
    uint32_t bound = 0;
    FrzScoreHist hist;
    FRZ_TRY(match_into_device(m, cs, index_offset, reversed, &d_list, &bound, stream, st, will_sort ? nullptr : final_out,
                              will_sort ? &hist : nullptr, scope));
    // `!self.patterns.is_empty() && sort.is_by_score()` (src/matcher/mod.rs:218)
    if (will_sort) {
        FrzMatchDev* other = final_out ? final_out : (d_list == ws.matches_a.get() ? ws.matches_b.get() : ws.matches_a.get());
        // two-pass sort (score bound >= 1024) needs a scratch list of the corpus size: the multi-pattern ping-pong
        // buffer is free at this point (d_list is never multi_a); grow it whenever THIS corpus is larger
        FrzMatchDev* tmp = nullptr;
        if (bound >= 1024) {
            FRZ_TRY(ensure_multi_buffers(m, cs.n));
            tmp = ws.multi_a.get();
        }
        if (hist.counts) FRZ_TRY(frz_launch_sort_fused(d_list, other, &ws.counters.get()->total, hist, ws.sort, stream, st, limit));
        else FRZ_TRY(frz_launch_sort_by_score_dev(d_list, tmp, other, &ws.counters.get()->total, bound, ws.sort, stream, st, limit));
        m->last_sort_bins = frz_sort_single_pass_bins(bound);
        d_list = other;
    } else if (final_out && d_list != final_out) {
        k_copy_n<<<grid_for(std::min<uint64_t>(cs.n, limit), 256), 256, 0, stream>>>(d_list, final_out, &ws.counters.get()->total, limit);
        st->launches++;
        d_list = final_out;
    }
    record_ev(ws, 3, stream);
    *d_result = d_list;
    return FRZ_OK;
}

}  // namespace
void collect_timings(frz_matcher* m, const FrzLaunchStats& st) {
    FrzWorkspace& ws = m->ws;
    float a = 0, b = 0, c = 0, t = 0;
    const bool* r = ws.ev_rec;
    if (r[0] && r[1] && cudaEventElapsedTime(&a, ws.ev[0].get(), ws.ev[1].get()) != cudaSuccess) a = 0;
    if (r[1] && r[2] && cudaEventElapsedTime(&b, ws.ev[1].get(), ws.ev[2].get()) != cudaSuccess) b = 0;
    if (r[2] && r[3] && cudaEventElapsedTime(&c, ws.ev[2].get(), ws.ev[3].get()) != cudaSuccess) c = 0;
    if (r[0] && r[3] && cudaEventElapsedTime(&t, ws.ev[0].get(), ws.ev[3].get()) != cudaSuccess) t = 0;
    cudaGetLastError();
    m->last_ms[0] = a; m->last_ms[1] = b; m->last_ms[2] = c; m->last_ms[3] = t;
    m->last_launches = st.launches;
}
namespace {

// The first min(limit, total) matches of d_list → host (a top-K call passes cap = limit, so it never fails on capacity);
// *n_out = their number, *n_total = all matches.
frz_status copy_out(frz_matcher* m, FrzMatchDev* d_list, uint64_t limit, frz_match* out, uint64_t cap, uint64_t* n_out,
                    uint64_t* n_total, cudaStream_t stream) {
    FRZ_TRY(read_counters(m, stream));
    const uint64_t total = m->ws.h_counters.get()->total;
    const uint64_t n = std::min(limit, total);
    if (n_out) *n_out = n;
    if (n_total) *n_total = total;
    if (n > cap) return frz_fail(FRZ_ERR_CAPACITY, "output capacity %llu < %llu matches", (unsigned long long)cap, (unsigned long long)n);
    if (n) {
        if (!out) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
        static_assert(sizeof(frz_match) == sizeof(FrzMatchDev), "layout");
        FRZ_CUDA_TRY(cudaMemcpyAsync(out, d_list, n * sizeof(frz_match), cudaMemcpyDeviceToHost, stream));
        FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    }
    return FRZ_OK;
}

// Matcher::match_list (into, from index_offset, in `sort` order) → host, truncated to its first `limit` rows (top-K calls:
// the same pipeline with a limit on the final scatter and copy; UINT64_MAX for the whole list).  scope: the rows of a subset
// call (match_into_device).
frz_status match_list_host(frz_matcher* m, const frz_corpus* corpus, uint32_t index_offset, uint8_t sort, uint64_t limit,
                           const SubsetScope& scope, frz_match* out, uint64_t cap, uint64_t* n_out, uint64_t* n_total) {
    if (scope.none) {
        if (n_out) *n_out = 0;
        if (n_total) *n_total = 0;
        return FRZ_OK;
    }
    cudaStream_t stream = nullptr;
    FrzLaunchStats st;
    FrzMatchDev* d_list = nullptr;
    const uint32_t dev_limit = (uint32_t)std::min<uint64_t>(limit, kFrzNoLimit);   // a list never holds more than 2^32 - 1 matches
    frz_status s = FRZ_OK;
    for (int attempt = 0; attempt < 2; attempt++) {
        s = match_list_device(m, corpus->st, index_offset, sort, &d_list, stream, &st, nullptr, dev_limit, scope);
        if (s == FRZ_OK) s = copy_out(m, d_list, limit, out, cap, n_out, n_total, stream);
        if (s != kRetryOverflow) break;
        FRZ_TRY(ensure_workspace(m, corpus->st, std::max<uint64_t>(corpus->st.n, 1)));  // worst-case lists, then once more
    }
    if (s == kRetryOverflow) s = frz_fail(FRZ_ERR_CUDA, "survivor list overflow persisted");
    collect_timings(m, st);
    return s;
}

}  // namespace

extern "C" frz_status frz_match_list(frz_matcher* m, const frz_corpus* corpus, frz_match* out, uint64_t cap, uint64_t* n_out) {
    if (!m || !corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_ensure_device(corpus->st.device));
    return match_list_host(m, corpus, 0, m->config.sort, UINT64_MAX, SubsetScope(), out, cap, n_out, nullptr);
}

extern "C" frz_status frz_match_list_top(frz_matcher* m, const frz_corpus* corpus, uint64_t k, frz_match* out, uint64_t* n_out,
                                         uint64_t* n_total) {
    if (!m || !corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    FRZ_TRY(frz_ensure_device(corpus->st.device));
    return match_list_host(m, corpus, 0, m->config.sort, k, SubsetScope(), out, k, n_out, n_total);
}

// ---------------------------------------------------------------------------------- subsets
// A bitmap over the indices [0, n_bits) of the corpus at creation (later appends lie beyond it and are not members), and
// the same members as an ascending list.
struct frz_subset {
    const frz_corpus* corpus;
    FrzDevArray<uint32_t> bits;      // ceil(n_bits / 32) words on the corpus's device (masked form)
    FrzDevArray<uint32_t> members;   // n_members ascending indices on the corpus's device (list form)
    uint64_t n_bits;
    uint64_t n_members;              // distinct members
};

extern "C" frz_status frz_subset_create(const frz_corpus* c, const uint32_t* which, uint64_t n, frz_subset** out) {
    if (!c || !out || (n && !which)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(check_indices(c, which, n));
    auto s = std::make_unique<frz_subset>();
    s->corpus = c;
    s->n_bits = c->st.n;
    std::vector<uint32_t> bits((s->n_bits + 31) / 32, 0);
    for (uint64_t j = 0; j < n; j++) bits[which[j] >> 5] |= 1u << (which[j] & 31);
    std::vector<uint32_t> members;
    for (size_t w = 0; w < bits.size(); w++)
        for (uint32_t x = bits[w]; x; x &= x - 1) members.push_back((uint32_t)(w * 32 + __builtin_ctz(x)));
    s->n_members = members.size();
    if (!bits.empty()) {
        FRZ_TRY(frz_ensure_device(c->st.device));
        FRZ_TRY(s->bits.reserve(bits.size()));
        FRZ_CUDA_TRY(cudaMemcpy(s->bits.get(), bits.data(), bits.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    if (!members.empty()) {
        FRZ_TRY(s->members.reserve(members.size()));
        FRZ_CUDA_TRY(cudaMemcpy(s->members.get(), members.data(), members.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    *out = s.release();
    return FRZ_OK;
}
extern "C" uint64_t frz_subset_len(const frz_subset* s) { return s ? s->n_members : 0; }
extern "C" void frz_subset_destroy(frz_subset* s) { delete s; }

// A subset call takes the list form when its members are at most FRZ_SUBSET_LIST_PERMILLE / 1000 of the corpus, the masked
// form otherwise (DESIGN.md §4.9: the threshold comes from tools/bench_subset.py).  Comparison builds set -1 (masked form
// only) or 1000 (list form only): `python frizbee_b200/build.py --variant NAME --define FRZ_SUBSET_LIST_PERMILLE=V`.
#ifndef FRZ_SUBSET_LIST_PERMILLE
#define FRZ_SUBSET_LIST_PERMILLE 20
#endif

namespace {
frz_status check_subset_call(const frz_matcher* m, const frz_corpus* corpus, const frz_subset* s) {
    if (!m || !corpus || !s) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (s->corpus != corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "the subset was made on another corpus");
    return frz_ensure_device(corpus->st.device);
}

// The rows of a subset call, built in the matcher's workspace on every call, so edits of the corpus between calls need no
// bookkeeping.  Masked form: the corpus's slot metadata with every non-member an unused slot.  List form: the members
// whose slots are in use, index-ordered.  An empty corpus keeps the default scope: it has no row.
frz_status subset_scope(frz_matcher* m, const frz_corpus* corpus, const frz_subset& s, cudaStream_t stream, SubsetScope* out) {
    const FrzCorpusStorage& cs = corpus->st;
    *out = SubsetScope();
    if (cs.n == 0) return FRZ_OK;
    FrzWorkspace& ws = m->ws;
    FRZ_TRY(ensure_workspace(m, cs, 0));   // (on this device; the lists are sized by the match call)
    constexpr int kListPermille = FRZ_SUBSET_LIST_PERMILLE;
    if (kListPermille >= 0 && s.n_members * 1000 <= cs.n * (uint64_t)std::max(kListPermille, 0)) {
        const uint64_t n = s.n_members;
        if (n == 0) { out->none = true; return FRZ_OK; }
        FRZ_TRY(ws.subset_list.reserve(2 * n));
        FrzMatchDev* tmp = ws.subset_list.get();
        FrzMatchDev* list = tmp + n;
        FRZ_CUDA_TRY(cudaMemsetAsync(ws.counters.get(), 0, sizeof(FrzCounters), stream));
        FrzLaunchStats uncounted;   // (the launches of a call are those of its pipeline)
        FRZ_TRY(retain_rows(m, LiveMember{s.members.get(), cs.slot_meta.get(), cs.slot_of.get(), tmp}, tmp, n, list, stream, &uncounted));
        FRZ_TRY(read_counters(m, stream));
        out->list = list;
        out->n_list = ws.h_counters.get()->total;
        out->none = out->n_list == 0;
        return FRZ_OK;
    }
    const uint64_t n_slots = (uint64_t)cs.n_tiles * FRZ_TILE;
    FRZ_TRY(ws.subset_meta.reserve(n_slots));
    k_subset_meta<<<grid_for(n_slots / 4, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(cs.slot_meta.get()), n_slots / 4,
                                                                  s.bits.get(), s.n_bits, reinterpret_cast<uint4*>(ws.subset_meta.get()));
    FRZ_CUDA_TRY(cudaGetLastError());
    out->masked_meta = ws.subset_meta.get();
    return FRZ_OK;
}
}  // namespace

extern "C" frz_status frz_match_list_subset(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, frz_match* out, uint64_t cap,
                                            uint64_t* n_out) {
    FRZ_TRY(check_subset_call(m, corpus, s));
    SubsetScope scope;
    FRZ_TRY(subset_scope(m, corpus, *s, nullptr, &scope));
    return match_list_host(m, corpus, 0, m->config.sort, UINT64_MAX, scope, out, cap, n_out, nullptr);
}

extern "C" frz_status frz_match_list_subset_top(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, uint64_t k, frz_match* out,
                                                uint64_t* n_out, uint64_t* n_total) {
    FRZ_TRY(check_subset_call(m, corpus, s));
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    SubsetScope scope;
    FRZ_TRY(subset_scope(m, corpus, *s, nullptr, &scope));
    return match_list_host(m, corpus, 0, m->config.sort, k, scope, out, k, n_out, n_total);
}

extern "C" frz_status frz_match_list_into(frz_matcher* m, const frz_corpus* corpus, uint32_t index_offset, frz_match* out,
                                          uint64_t cap, uint64_t* n_out) {
    if (!m || !corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_ensure_device(corpus->st.device));
    return match_list_host(m, corpus, index_offset, FRZ_SORT_INDEX_ASC, UINT64_MAX, SubsetScope(), out, cap, n_out, nullptr);
}

namespace {   // defined with the shard calls below
bool streamed_eligible(const frz_matcher* m, uint64_t n, uint32_t index_offset);
frz_status match_streamed_impl(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n, int device,
                               uint32_t index_offset, FrzMatchDev* d_out, uint64_t* d_count, cudaStream_t stream, FrzMatchDev** d_result);
}  // namespace

// End to end from host Arrow buffers: streamed H2D + pack (pack.cu: ingest_host_t), match, D2H of the matches.
extern "C" frz_status frz_match_list_host_arrow(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n,
                                                int device, frz_match* out, uint64_t cap, uint64_t* n_out) {
    if (!m || !offsets) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_check_offset_width(offset_width));
    if (n > 0xFFFFFFFFull) return frz_fail(FRZ_ERR_TOO_MANY_ITEMS, "too many items in haystack: %llu", (unsigned long long)n);
    if (streamed_eligible(m, n, 0)) {   // the match pipeline runs while the list streams in (frz_match_shard_streamed)
        FrzMatchDev* d_list = nullptr;
        FRZ_TRY(match_streamed_impl(m, bytes, offsets, offset_width, n, device, 0, nullptr, nullptr, nullptr, &d_list));
        const frz_status s = copy_out(m, d_list, UINT64_MAX, out, cap, n_out, nullptr, nullptr);
        m->timings_pending = false;
        FrzLaunchStats st; st.launches = m->last_launches;
        collect_timings(m, st);
        return s;
    }
    const frz_corpus* c = nullptr;
    FRZ_TRY(frz_matcher_ingest_e2e(m, bytes, offsets, offset_width, n, device, &c));
    return frz_match_list(m, c, out, cap, n_out);
}

namespace {
// The matcher's end-to-end staging arena and packed corpus, for `device`: emptied first when they live on another device.
frz_corpus& e2e_corpus_on(frz_matcher* m, int device) {
    if (m->e2e_corpus.st.device != device) {
        m->e2e_ingest = FrzIngest();
        m->e2e_corpus.st = FrzCorpusStorage();
        m->e2e_corpus.st.device = device;
    }
    return m->e2e_corpus;
}
}  // namespace

// The ingest half of the end-to-end call: host Arrow buffers → the matcher's reusable packed corpus (grow-only staging
// arena, streamed H2D overlapped with the pack kernels; asynchronous on the legacy default stream).
frz_status frz_matcher_ingest_e2e(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n, int device,
                                  const frz_corpus** out) {
    if (!m || !offsets || !out) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_check_offset_width(offset_width));
    if (n > 0xFFFFFFFFull) return frz_fail(FRZ_ERR_TOO_MANY_ITEMS, "too many items in haystack: %llu", (unsigned long long)n);
    FRZ_TRY(frz_ensure_device(device));
    cudaStream_t stream = nullptr;
    frz_corpus& c = e2e_corpus_on(m, device);
    FRZ_TRY(frz_ingest_host(m->e2e_ingest, bytes, offsets, offset_width, n, stream, &c.st));
    *out = &c;
    return FRZ_OK;
}

extern "C" frz_status frz_match_list_host(frz_matcher* m, const uint8_t* bytes, const uint64_t* offsets, uint64_t n, int device,
                                          frz_match* out, uint64_t cap, uint64_t* n_out) {
    return frz_match_list_host_arrow(m, bytes, offsets, 8, n, device, out, cap, n_out);
}

// Matcher::match_list_indices for chosen haystacks (src/matcher/mod.rs:234-262): Match + matched byte offsets.
namespace {
// one pattern over the chosen rows: match_one_indices_impl (fuzzy / literal), results in host arrays
frz_status match_indices_one(const Compiled& c, const frz_corpus* corpus, const uint32_t* which, uint64_t n, frz_match* out_matches,
                             uint32_t* out_indices, uint32_t stride, uint32_t* out_counts) {
    cudaStream_t stream = nullptr;
    const uint32_t threads = (uint32_t)std::min<uint64_t>(n, 1024);
    const int rows = c.unicode ? c.un.n : c.un.nbytes;
    const uint64_t sstride = c.literal ? 1 : (uint64_t)frzi::indices_scratch_elems(rows, c.dev.sw_lanes);
    FrzDevArray<uint32_t> d_which, d_idx, d_cnt;
    FrzDevArray<FrzMatchDev> d_m;
    FrzDevArray<uint16_t> d_scratch;
    FRZ_TRY(d_which.reserve(n));
    FRZ_TRY(d_idx.reserve(n * (uint64_t)stride));
    FRZ_TRY(d_cnt.reserve(n));
    FRZ_TRY(d_m.reserve(n));
    FRZ_TRY(d_scratch.reserve((uint64_t)threads * sstride));
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_which.get(), which, n * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
    FRZ_CUDA_TRY(cudaMemsetAsync(d_m.get(), 0, n * sizeof(FrzMatchDev), stream));
    FRZ_TRY(frz_launch_match_indices(corpus->st.view(), c.dev, c.un, c.usc, c.unicode, d_which.get(), n, d_m.get(), d_idx.get(), stride,
                                     d_cnt.get(), d_scratch.get(), sstride, threads, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(out_matches, d_m.get(), n * sizeof(FrzMatchDev), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(out_indices, d_idx.get(), n * (uint64_t)stride * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(out_counts, d_cnt.get(), n * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    return FRZ_OK;
}

__global__ void k_rows_removed(const uint32_t* __restrict__ slot_meta, const uint16_t* __restrict__ slot_of, const uint32_t* __restrict__ which,
                               uint64_t n, uint64_t corpus_n, uint8_t* __restrict__ removed) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t idx = which[j];
        removed[j] = idx < corpus_n && !slot_in_use(slot_meta, slot_of, idx);
    }
}

// removed[j] = haystack which[j] was removed (frz_corpus_remove)
frz_status rows_removed(const frz_corpus* corpus, const uint32_t* which, uint64_t n, uint8_t* removed) {
    cudaStream_t stream = nullptr;
    FrzDevArray<uint32_t> d_which;
    FrzDevArray<uint8_t> d_removed;
    FRZ_TRY(d_which.reserve(n));
    FRZ_TRY(d_removed.reserve(n));
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_which.get(), which, n * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
    k_rows_removed<<<grid_for(n, 256), 256, 0, stream>>>(corpus->st.slot_meta.get(), corpus->st.slot_of.get(), d_which.get(), n, corpus->st.n,
                                                      d_removed.get());
    FRZ_CUDA_TRY(cudaGetLastError());
    FRZ_CUDA_TRY(cudaMemcpyAsync(removed, d_removed.get(), n, cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    return FRZ_OK;
}
}  // namespace

extern "C" frz_status frz_match_indices(frz_matcher* m, const frz_corpus* corpus, const uint32_t* which, uint64_t n,
                                        frz_match* out_matches, uint32_t* out_indices, uint32_t stride, uint32_t* out_counts) {
    if (!m || !corpus || (n && (!which || !out_matches || !out_indices || !out_counts)) || stride == 0)
        return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (m->compiled.empty()) return frz_fail(FRZ_ERR_INVALID_ARG, "the matcher has no pattern");
    for (const Compiled& c : m->compiled)   // the indices kernel keeps per-needle-byte state in arrays of FRZ_MAX_NEEDLE
        if (c.is_long())
            return frz_fail(FRZ_ERR_UNSUPPORTED, "match_indices handles needles of up to %d bytes (this one has %d)", FRZ_MAX_NEEDLE, c.dev.n);
    if (n == 0) return FRZ_OK;
    FRZ_TRY(frz_ensure_device(corpus->st.device));
    if (m->compiled.size() == 1 && !m->compiled[0].negated)   // CompiledPatterns::Single
        return match_indices_one(m->compiled[0], corpus, which, n, out_matches, out_indices, stride, out_counts);
    // CompiledPatterns::Multi → match_one_indices_multi (src/matcher/multi.rs:56-79): a negated atom that matches drops the
    // row, the others add their scores, OR their exact flags and pool their indices (sorted descending, de-duplicated)
    // every atom yields at most one index per needle scalar (<= FRZ_MAX_NEEDLE): pool with an internal stride that
    // cannot truncate an atom, cut the pooled (sorted, de-duplicated) list at the caller's stride afterwards
    const uint32_t istride = std::max<uint32_t>(stride, FRZ_MAX_NEEDLE);
    std::vector<frz_match> pm(n);
    std::vector<uint32_t> pi((size_t)n * istride), pc(n);
    std::vector<std::vector<uint32_t>> pooled(n);
    std::vector<uint8_t> alive(n, 1);
    if (corpus->st.n_removed) {   // an all-negated matcher would keep a removed row: none of its atoms can hit it
        std::vector<uint8_t> removed(n);
        FRZ_TRY(rows_removed(corpus, which, n, removed.data()));
        for (uint64_t j = 0; j < n; j++) alive[j] = !removed[j];
    }
    for (uint64_t j = 0; j < n; j++) out_matches[j] = frz_match{which[j], 0, 0, 0};
    for (const Compiled& c : m->compiled) {
        FRZ_TRY(match_indices_one(c, corpus, which, n, pm.data(), pi.data(), istride, pc.data()));
        for (uint64_t j = 0; j < n; j++) {
            if (!alive[j]) continue;
            const bool hit = pc[j] != 0xFFFFFFFFu;
            if (c.negated) { if (hit) alive[j] = 0; continue; }
            if (!hit) { alive[j] = 0; continue; }
            const uint32_t sum = (uint32_t)out_matches[j].score + pm[j].score;
            out_matches[j].score = (uint16_t)std::min<uint32_t>(sum, 0xFFFF);
            out_matches[j].exact |= pm[j].exact;
            const size_t got = std::min<size_t>(pc[j], istride);
            pooled[j].insert(pooled[j].end(), pi.begin() + (size_t)j * istride, pi.begin() + (size_t)j * istride + got);
        }
    }
    for (uint64_t j = 0; j < n; j++) {
        if (!alive[j]) { out_counts[j] = 0xFFFFFFFFu; continue; }
        auto& v = pooled[j];
        std::sort(v.begin(), v.end(), [](uint32_t a, uint32_t b) { return a > b; });
        v.erase(std::unique(v.begin(), v.end()), v.end());
        out_counts[j] = (uint32_t)v.size();   // untruncated: a value > stride tells the caller the row was cut
        for (uint32_t k = 0; k < std::min<uint32_t>(out_counts[j], stride); k++) out_indices[(size_t)j * stride + k] = v[k];
    }
    return FRZ_OK;
}

extern "C" frz_status frz_match_shard_device(frz_matcher* m, const frz_corpus* shard, uint32_t index_offset, frz_match* d_out,
                                             uint64_t cap, uint64_t* d_count, void* stream_) {
    return frz_match_shard_device_top(m, shard, index_offset, d_out, cap, d_count, stream_, kFrzNoLimit);
}

// frz_match_shard_device whose run holds only its first `limit` elements (the count is still the full match count)
frz_status frz_match_shard_device_top(frz_matcher* m, const frz_corpus* shard, uint32_t index_offset, frz_match* d_out, uint64_t cap,
                                      uint64_t* d_count, void* stream_, uint32_t limit) {
    if (!m || !shard || !d_out || !d_count) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_ensure_device(shard->st.device));
    cudaStream_t stream = (cudaStream_t)stream_;
    // asynchronous entry point: nobody reads the overflow flag back, so size the lists for the worst case
    FRZ_TRY(ensure_workspace(m, shard->st, std::max<uint64_t>(shard->st.n, 1)));
    // the run can never exceed the shard size; the caller sizes d_out as >= shard length
    if (cap < shard->st.n) return frz_fail(FRZ_ERR_CAPACITY, "d_out must hold the whole shard (%llu)", (unsigned long long)shard->st.n);
    // (the count of a multi-pattern or empty matcher exists only at the end)
    return shard_call(m, d_count, stream, [&](FrzLaunchStats* st) {
        FrzMatchDev* d_list = nullptr;
        return match_list_device(m, shard->st, index_offset, m->config.sort, &d_list, stream, st, reinterpret_cast<FrzMatchDev*>(d_out),
                                 limit);
    });
}

// Makes `stream` wait until the count of the last frz_match_shard_device call has been written to its d_count
// (which happens before the scoring kernels for a single-pattern matcher).
extern "C" frz_status frz_matcher_wait_count(frz_matcher* m, void* stream) {
    if (!m) return frz_fail(FRZ_ERR_INVALID_ARG, "null matcher");
    if (!m->count_ev) return frz_fail(FRZ_ERR_INVALID_ARG, "no shard call has been made on this matcher");
    FRZ_CUDA_TRY(cudaStreamWaitEvent((cudaStream_t)stream, m->count_ev.get(), 0));
    return FRZ_OK;
}

// ---- streamed shard call: host Arrow buffers in, locally ordered run out, the match pipeline overlapped with the H2D copy ----
// The tiles of a packed corpus are independent, so the pipeline can run on tiles [t0, t1) through a SUB-VIEW of the corpus
// (array pointers advanced to tile t0; unit addresses are absolute) as soon as their H2D chunk has been packed: length gate →
// signature scan → exact windows → tile scan (carrying the running match count, so every range appends to the same
// index-ordered list) → scoring.  Only the score sort waits for the last chunk.  The copy engine stays busy from the first
// byte to the last; what is left after the last chunk lands is one range's pipeline + the sort instead of the whole list's.
namespace {
struct StreamedCtx {
    frz_matcher* m;
    const Compiled* c;
    uint32_t index_offset;
    FrzMatchDev* dst;       // index-ordered matches (pre-sort)
    const FrzNeedleTab* ntab;   // the needle table of a long needle (uploaded before the ingest starts), else nullptr
    cudaStream_t stream;
    FrzLaunchStats* st;
    uint32_t pending_t0;    // first tile not yet matched
    int chunks_pending;     // packed chunks since the last range
    int group;              // chunks per range
};
frz_status streamed_range(StreamedCtx& x, uint32_t t0, uint32_t t1, bool last) {
    frz_matcher* m = x.m;
    FrzWorkspace& ws = m->ws;
    const FrzCorpusStorage& cs = m->e2e_corpus.st;
    FrzCorpusView cv = cs.view();
    cv.tile_base += t0;
    cv.groups += (size_t)t0 * FRZ_GROUPS_PER_TILE;
    cv.slot_meta += (size_t)t0 * FRZ_TILE;
    cv.slot_of += (size_t)t0 * FRZ_TILE;
    cv.slot_sig += (size_t)t0 * FRZ_TILE;
    cv.n = std::min<uint64_t>(cs.n, (uint64_t)t1 * FRZ_TILE) - (uint64_t)t0 * FRZ_TILE;
    cv.n_tiles = t1 - t0;
    const uint32_t off = x.index_offset + t0 * FRZ_TILE;
    FRZ_CUDA_TRY(cudaMemsetAsync(ws.counters.get(), 0, sizeof(FrzCounters), x.stream));
    FRZ_TRY(frz_launch_prefilter(cv, x.c->dev, ws, x.stream, x.st, x.ntab));
    FRZ_TRY(frz_launch_tile_scan(cv, ws, x.stream, x.st, ws.stream_total.get()));
    if (last) {
        record_ev(ws, 1, x.stream);
        // the running count is final: publish it before the last range is scored
        if (m->early_count_dst) FRZ_TRY(publish_count(m, m->early_count_dst, x.stream));
    }
    FRZ_TRY(frz_launch_sw(cv, x.c->dev, off, false, ws, x.dst, x.stream, x.st, FrzScoreHist(), x.ntab));
    return FRZ_OK;
}
frz_status streamed_after_chunk(void* ctx, uint32_t t0, uint32_t t1, bool last) {
    StreamedCtx& x = *static_cast<StreamedCtx*>(ctx);
    (void)t0;
    x.chunks_pending++;
    if (!last && x.chunks_pending < x.group) return FRZ_OK;
    const uint32_t r0 = x.pending_t0;
    x.pending_t0 = t1;
    x.chunks_pending = 0;
    if (t1 <= r0) return FRZ_OK;
    return streamed_range(x, r0, t1, last);
}
}  // namespace

namespace {
bool streamed_eligible(const frz_matcher* m, uint64_t n, uint32_t index_offset) {
    const uint8_t sort = m->config.sort;
    return m->compiled.size() == 1 && !m->compiled[0].negated && !m->compiled[0].unicode &&
           (sort == FRZ_SORT_INDEX_ASC || sort == FRZ_SORT_SCORE_THEN_INDEX_ASC) &&   // reversed lists need the final total per element
           n >= 64 * FRZ_TILE && (uint64_t)n + index_offset <= 0xFFFFFFFFull;
}
}  // namespace
// (match_streamed_impl: d_out == nullptr leaves the list in the matcher's own buffer, returned through d_result;
//  d_count == nullptr uses a spare device slot)

frz_status frz_match_shard_streamed(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n, int device,
                                    uint32_t index_offset, frz_match* d_out, uint64_t cap, uint64_t* d_count, void* stream_) {
    if (!m || !offsets || !d_out || !d_count) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_check_offset_width(offset_width));
    if (!streamed_eligible(m, n, index_offset)) {
        const frz_corpus* shard = nullptr;
        FRZ_TRY(frz_matcher_ingest_e2e(m, bytes, offsets, offset_width, n, device, &shard));
        return frz_match_shard_device(m, shard, index_offset, d_out, cap, d_count, stream_);
    }
    if (cap < n) return frz_fail(FRZ_ERR_CAPACITY, "d_out must hold the whole shard (%llu)", (unsigned long long)n);
    return match_streamed_impl(m, bytes, offsets, offset_width, n, device, index_offset, reinterpret_cast<FrzMatchDev*>(d_out), d_count,
                               (cudaStream_t)stream_, nullptr);
}

namespace {
frz_status match_streamed_impl(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n, int device,
                               uint32_t index_offset, FrzMatchDev* d_out, uint64_t* d_count, cudaStream_t stream, FrzMatchDev** d_result) {
    const uint8_t sort = m->config.sort;
    FRZ_TRY(frz_ensure_device(device));
    frz_corpus& c = e2e_corpus_on(m, device);
    c.st.n = n;
    c.st.n_tiles = (uint32_t)((n + FRZ_TILE - 1) / FRZ_TILE);
    FrzWorkspace& ws = m->ws;
    FRZ_TRY(ensure_workspace(m, c.st, std::max<uint64_t>(n, 1)));   // nobody reads the overflow flag back: worst-case lists
    const Compiled& pat = m->compiled[0];
    const bool will_sort = sort == FRZ_SORT_SCORE_THEN_INDEX_ASC;
    FrzMatchDev* final_out = d_out ? d_out : ws.matches_b.get();
    if (!d_count) d_count = reinterpret_cast<uint64_t*>(ws.stream_total.get() + 1);
    if (d_result) *d_result = final_out;
    return shard_call(m, d_count, stream, [&](FrzLaunchStats* st) -> frz_status {
        reset_call_state(m);
        StreamedCtx x;
        x.m = m; x.c = &pat; x.index_offset = index_offset; x.dst = will_sort ? ws.matches_a.get() : final_out; x.stream = stream; x.st = st;
        FRZ_TRY(needle_table(m, pat, &x.ntab));   // a synchronous upload, so before the first H2D chunk
        x.pending_t0 = 0; x.chunks_pending = 0;
        x.group = 4;   // a range per four H2D chunks (about 1/8 of the list): the tail after the last chunk is one range + the sort
        FRZ_CUDA_TRY(cudaMemsetAsync(ws.stream_total.get(), 0, sizeof(unsigned long long), stream));
        record_ev(ws, 0, stream);
        FRZ_TRY(frz_ingest_host(m->e2e_ingest, bytes, offsets, offset_width, n, stream, &c.st, streamed_after_chunk, &x));
        record_ev(ws, 2, stream);
        if (will_sort) {
            FrzMatchDev* tmp = nullptr;
            if (pat.score_bound >= 1024) { FRZ_TRY(ensure_multi_buffers(m, n)); tmp = ws.multi_a.get(); }
            FRZ_TRY(frz_launch_sort_by_score_dev(ws.matches_a.get(), tmp, final_out, &ws.counters.get()->total, pat.score_bound, ws.sort, stream, st));
            m->last_sort_bins = frz_sort_single_pass_bins(pat.score_bound);
        }
        record_ev(ws, 3, stream);
        return FRZ_OK;
    });
}
}  // namespace

// Debugging / test aid: the compiled device pattern of pattern i (the struct the kernels receive), so that host
// builds of the kernel cores (tests/test_kernel_logic_cpu.py) run with exactly the constants the GPU gets.
extern "C" frz_status frz_matcher_debug_pattern(const frz_matcher* m, size_t i, void* out, size_t out_size) {
    if (!m || !out || i >= m->compiled.size()) return frz_fail(FRZ_ERR_INVALID_ARG, "pattern index out of range");
    if (out_size != sizeof(FrzPatternDev)) return frz_fail(FRZ_ERR_INVALID_ARG, "expected a buffer of %zu bytes", sizeof(FrzPatternDev));
    memcpy(out, &m->compiled[i].dev, sizeof(FrzPatternDev));
    return FRZ_OK;
}

// Debugging / test aid: the needle and scoring constants pattern i hands to the unicode, literal and traceback kernels
// (k_unicode, k_match_indices), so that host builds of unicode_path.cuh / indices_path.cuh run with exactly them.
extern "C" frz_status frz_matcher_debug_unicode(const frz_matcher* m, size_t i, void* un, size_t un_size, void* usc, size_t usc_size) {
    if (!m || !un || !usc || i >= m->compiled.size()) return frz_fail(FRZ_ERR_INVALID_ARG, "pattern index out of range");
    if (un_size != sizeof(FrzUNeedle) || usc_size != sizeof(FrzUScoring))
        return frz_fail(FRZ_ERR_INVALID_ARG, "expected buffers of %zu and %zu bytes", sizeof(FrzUNeedle), sizeof(FrzUScoring));
    memcpy(un, &m->compiled[i].un, sizeof(FrzUNeedle));
    memcpy(usc, &m->compiled[i].usc, sizeof(FrzUScoring));
    return FRZ_OK;
}

extern "C" uint64_t frz_debug_device_bytes(void) { return g_frz_device_bytes.load(); }
extern "C" uint64_t frz_debug_device_bytes_peak(int reset) {
    if (reset) g_frz_device_bytes_peak.store(g_frz_device_bytes.load());
    return g_frz_device_bytes_peak.load();
}

extern "C" uint32_t frz_matcher_score_bound(const frz_matcher* m) {
    if (!m) return 0;
    uint64_t b = 0;
    for (const auto& c : m->compiled) if (!c.negated) b += c.score_bound;
    return (uint32_t)std::min<uint64_t>(b, 0xFFFF);
}

extern "C" frz_status frz_radix_sort_matches(frz_match* matches, uint64_t n, int device) {
    if (n == 0) return FRZ_OK;
    if (!matches) return frz_fail(FRZ_ERR_INVALID_ARG, "null matches");
    FRZ_TRY(frz_ensure_device(device));
    FrzDevArray<FrzMatchDev> d_a, d_b, d_c;
    FrzDevArray<unsigned long long> d_n;
    FrzSortScratch ss;
    cudaStream_t stream = nullptr;
    FRZ_TRY(d_a.reserve(n));
    FRZ_TRY(d_b.reserve(n));
    FRZ_TRY(d_c.reserve(n));
    FRZ_TRY(d_n.reserve(1));
    FRZ_TRY(frz_sort_hist_alloc(ss.hist));
    unsigned long long hn = n;
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_n.get(), &hn, sizeof hn, cudaMemcpyHostToDevice, stream));
    FRZ_CUDA_TRY(cudaMemcpyAsync(d_a.get(), matches, n * sizeof(FrzMatchDev), cudaMemcpyHostToDevice, stream));
    FRZ_TRY(frz_launch_sort_by_score_dev(d_a.get(), d_b.get(), d_c.get(), d_n.get(), 0xFFFF, ss, stream, nullptr));
    FRZ_CUDA_TRY(cudaMemcpyAsync(matches, d_c.get(), n * sizeof(FrzMatchDev), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    return FRZ_OK;
}
