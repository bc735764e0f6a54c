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
#include <optional>

#include "batch_collapse_plan.cuh"
#include "batch_order_plan.cuh"
#include "batch_columns_plan.cuh"
#include "batch_plan.cuh"
#include "collapse_plan.cuh"
#include "frz_device.cuh"
#include "frz_host.h"
#include "unicode_needle.h"
#include "indices_path.cuh"
#include "where_plan.cuh"

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
// a list of frz_match_list_columns: retain the rows whose slot is in use in each of up to kLiveColumns further columns
// (the candidate-list kernels read a candidate's slot metadata unchecked, so a row removed in a later column must leave
// the list before that column is read)
constexpr int kLiveColumns = 8;
struct LiveInColumns {
    const FrzMatchDev* list;
    uint32_t index_offset;
    int n;
    const uint32_t* slot_meta[kLiveColumns];
    const uint16_t* slot_of[kLiveColumns];
    __device__ bool operator()(uint64_t i) const {
        const uint64_t idx = list[i].index - index_offset;
        for (int c = 0; c < n; c++)
            if (!slot_in_use(slot_meta[c], slot_of[c], idx)) return false;
        return true;
    }
};
// a collapsed call's list: retain the rows of C (collapse_plan.cuh), after the rounds
struct CollapseKeep {
    FrzCollapseDev c;
    const FrzMatchDev* list;
    __device__ bool operator()(uint64_t i) const {
        const uint32_t g = frz_collapse_group(c.ids, c.n_ids, list[i].index);
        return frz_collapse_keep(g, g == kFrzGroupNone ? 0u : c.counts[g], c.per_group, c.taken[i] != 0);
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

// A long needle's FrzNeedleTab on `device` (the device of the call's workspace, which is m's own unless m's pattern runs in
// another matcher's frz_match_list_columns call), uploaded once per compiled pattern set (build_patterns starts a new
// epoch) and device; nullptr for other needles.
frz_status needle_table(frz_matcher* m, const Compiled& c, int device, const FrzNeedleTab** out) {
    *out = nullptr;
    if (!c.is_long()) return FRZ_OK;
    if (!m->ntab.get() || m->ntab.device() != device || m->ntab_epoch != m->epoch) {
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
// read in place of the corpus's own, nullptr = the corpus's.  owner: the matcher whose pattern c is, when it is not m
// (frz_match_list_columns runs every column's patterns in ms[0]'s workspace).
frz_status run_pattern(frz_matcher* m, const FrzCorpusStorage& cs, const Compiled& c, const uint32_t* masked_meta,
                       uint32_t index_offset, bool reversed, FrzMatchDev* d_out, cudaStream_t stream, FrzLaunchStats* st,
                       bool record_events, const FrzMatchDev* cand_list = nullptr, uint64_t n_cand = 0,
                       const FrzScoreHist& hist = FrzScoreHist(), frz_matcher* owner = nullptr) {
    FrzWorkspace& ws = m->ws;
    FrzCorpusView cv = cs.view();
    if (masked_meta) cv.slot_meta = masked_meta;
    uint64_t cap = std::max(ws.survivor_cap(), initial_survivor_cap(cs, c.dev));
    FRZ_TRY(ensure_workspace(m, cs, cap));
    const FrzNeedleTab* ntab = nullptr;
    FRZ_TRY(needle_table(owner ? owner : m, c, ws.device, &ntab));
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

// One pattern of the multi-pattern loop (match_patterns) and the column it reads.  A matcher's own patterns all read the
// call's corpus; frz_match_list_columns gives each column's patterns their column.  owner: the matcher the compiled
// pattern belongs to (its long-needle table).
struct ColumnPattern {
    const Compiled* c;
    frz_matcher* owner;
    const FrzCorpusStorage* cs;
};

// The columns of a frz_match_list_columns call, as match_patterns takes them: every column's patterns in column order,
// the further columns with removed rows, and whether any matcher has a compiled pattern (the score sort's condition).
struct Columns {
    std::vector<ColumnPattern> pats;
    std::vector<const FrzCorpusStorage*> live;
    bool any_compiled = false;
};

// CompiledPatterns::Multi (src/matcher/multi.rs:84-152), each pattern over its own column; all columns share one index
// space and so one tile count.  The base, the first non-negated pattern, is scanned over its column, restricted to scope;
// every later pattern runs on the surviving candidates against its own column.  Without a base the list starts from every
// live row (or the scope's members).  cs: the base's column, else the column whose live rows start the list; scope is
// built against its slot metadata.  live: further columns with removed rows, whose removed rows leave the starting
// list before any later pattern reads it (LiveInColumns; empty for a matcher's own patterns).  Counts are read back
// between patterns.  The list lands in ws.matches_a (reversed if final_reversed), its count in ws.counters->total, and
// *score_bound is the saturating sum of the non-negated patterns' bounds.
frz_status match_patterns(frz_matcher* m, const std::vector<ColumnPattern>& pats, const FrzCorpusStorage& cs,
                          const std::vector<const FrzCorpusStorage*>& live, uint32_t index_offset, bool final_reversed,
                          FrzMatchDev** d_result, uint32_t* score_bound, cudaStream_t stream, FrzLaunchStats* st,
                          const SubsetScope& scope) {
    FrzWorkspace& ws = m->ws;
    const uint32_t* masked_meta = scope.masked_meta;
    FRZ_TRY(ensure_workspace(m, cs, pats.empty() ? 1 : initial_survivor_cap(cs, pats[0].c->dev)));
    FRZ_TRY(ensure_multi_buffers(m, cs.n));
    int base = -1;
    for (size_t i = 0; i < pats.size(); i++) if (!pats[i].c->negated) { base = (int)i; break; }
    FrzMatchDev* cand = ws.multi_a.get();
    FrzMatchDev* spare = ws.multi_b.get();
    uint64_t nc = 0;
    uint64_t bound = 0;
    if (base >= 0) {
        FRZ_TRY(run_pattern(m, cs, *pats[base].c, masked_meta, index_offset, false, cand, stream, st, true, scope.list, scope.n_list,
                            FrzScoreHist(), pats[base].owner));
        FRZ_TRY(read_counters(m, stream));
        nc = ws.h_counters.get()->total;
        bound = pats[base].c->score_bound;
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
    for (size_t c0 = 0; c0 < live.size() && nc > 0; c0 += kLiveColumns) {
        LiveInColumns rule{cand, index_offset, (int)std::min<size_t>(kLiveColumns, live.size() - c0), {}, {}};
        for (int c = 0; c < rule.n; c++) {
            rule.slot_meta[c] = live[c0 + c]->slot_meta.get();
            rule.slot_of[c] = live[c0 + c]->slot_of.get();
        }
        FRZ_TRY(retain_rows(m, rule, cand, nc, spare, stream, st));
        FRZ_TRY(read_counters(m, stream));
        nc = ws.h_counters.get()->total;
        std::swap(cand, spare);
    }
    FRZ_TRY(ensure_retain_buffers(m, cs.n));   // once, for every negated pattern below
    frz_status status = FRZ_OK;
    for (size_t pi = 0; pi < pats.size() && status == FRZ_OK; pi++) {
        if ((int)pi == base || nc == 0) continue;
        const Compiled& pat = *pats[pi].c;
        status = [&]() -> frz_status {
            // evaluate the pattern on the surviving candidates only, against its own column; hits land in ws.matches_a,
            // index-ordered, with real indices
            FRZ_TRY(run_pattern(m, *pats[pi].cs, pat, nullptr, index_offset, false, ws.matches_a.get(), stream, st, false, cand, nc,
                                FrzScoreHist(), pats[pi].owner));
            FRZ_TRY(read_counters(m, stream));
            const uint64_t nh = ws.h_counters.get()->total;
            if (pat.negated) {
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
                bound += pat.score_bound;
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
    // CompiledPatterns::Multi: every pattern over this corpus
    std::vector<ColumnPattern> cols;
    cols.reserve(pats.size());
    for (const Compiled& c : pats) cols.push_back(ColumnPattern{&c, m, &cs});
    return match_patterns(m, cols, cs, {}, index_offset, final_reversed, d_result, score_bound, stream, st, scope);
}

// Matcher::match_list on device: into (+reverse) (+stable score sort).  Result pointer + device count.
__global__ void k_copy_n(const FrzMatchDev* __restrict__ in, FrzMatchDev* __restrict__ out, const unsigned long long* n_ptr,
                         uint32_t limit) {
    const unsigned long long n = min(*n_ptr, (unsigned long long)limit);
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        out[i] = in[i];
}

// The boost of a ranked call (frz_match_list_ranked): the list is sorted by key = clamp(score + boost[index], 0, 65535).
struct Ranking {
    const int16_t* boost = nullptr;   // n values on the corpus's device; indices >= n have boost 0
    uint32_t n = 0;
    uint32_t max_boost = 0;           // >= every boost value (0 when none is positive): the key bound is score bound + this
};

// The groups of a collapsed call (frz_match_list_collapsed): of the list, only the rows of C (collapse_plan.cuh) are sorted
// and returned, and the list's rows per group are left in ws.collapse_counts.
struct Collapse {
    const uint32_t* ids = nullptr;    // group of index i < n_ids, on the corpus's device
    uint64_t n_ids = 0;
    uint64_t n_groups = 0;
    uint64_t per_group = 0;           // 1..kFrzCollapseMaxPerGroup, or UINT64_MAX: no cap (only the counts)
};

// The collapsed call's steps between the list and its sort (DESIGN.md §4.12): the count pass, per_group rounds, and the
// stable compaction of the kept rows into the other list buffer (*d_list then points there, and ws.counters->total holds
// |C|).  order: what the rows' order keys rank by.  ord (an ordered call's attribute, boost and order; `reversed` is set
// here): L is the ordered list, so the rounds rank by its 112-bit order key instead and `order` is not read.  The keys
// are computed into ws.order_keys in list order first (k_order_keys), and each round is collapse_plan.cuh's two-step max
// over them (DESIGN.md §4.15.1).  The list's length is read back first (a survivor-list overflow returns kRetryOverflow
// there): the passes and the compaction then cover the list, not the corpus.
frz_status collapse_list(frz_matcher* m, const FrzCorpusStorage& cs, const Collapse& col, uint8_t order, bool reversed,
                         const std::optional<Ranking>& rank, const FrzOrderDev* ord, FrzMatchDev** d_list, cudaStream_t stream,
                         FrzLaunchStats* st) {
    FrzWorkspace& ws = m->ws;
    FRZ_TRY(read_counters(m, stream));
    const uint64_t n_list = ws.h_counters.get()->total;
    const uint64_t n_cap = std::max<uint64_t>(cs.n, 1);
    FRZ_TRY(ws.collapse_counts.reserve(col.n_groups));
    if (ws.collapse_best.cap() < col.n_groups) {   // a new table starts zero; the rounds leave it zero
        FRZ_TRY(ws.collapse_best.reserve(col.n_groups));
        FRZ_CUDA_TRY(cudaMemsetAsync(ws.collapse_best.get(), 0, col.n_groups * sizeof(unsigned long long), stream));
    }
    FRZ_TRY(ws.collapse_taken.reserve(n_cap));
    const bool capped = col.per_group != UINT64_MAX;
    FrzCollapseDev c;
    c.ids = col.ids;
    c.n_ids = col.n_ids;
    c.boost = rank ? rank->boost : nullptr;
    c.n_boost = rank ? rank->n : 0;
    c.counts = ws.collapse_counts.get();
    c.best = ws.collapse_best.get();
    c.taken = ws.collapse_taken.get();
    c.per_group = capped ? (uint32_t)col.per_group : 0xFFFFFFFFu;
    c.order = order;
    c.reversed = reversed;
    const unsigned long long* n_ptr = &ws.counters.get()->total;
    if (ord && capped && n_list > 0) {
        if (ws.collapse_best_lo.cap() < col.n_groups) {   // as collapse_best
            FRZ_TRY(ws.collapse_best_lo.reserve(col.n_groups));
            FRZ_CUDA_TRY(cudaMemsetAsync(ws.collapse_best_lo.get(), 0, col.n_groups * sizeof(unsigned long long), stream));
        }
        FRZ_TRY(ws.order_keys.reserve(n_list));
        FRZ_TRY(ws.order_state.reserve(1));
        FrzOrderDev o = *ord;
        o.reversed = reversed;
        FRZ_TRY(frz_launch_order_keys(*d_list, n_ptr, n_list, o, ws.order_keys.get(), ws.order_state.get(), stream, st));
        FRZ_TRY(frz_launch_collapse_by_key(c, ws.collapse_best_lo.get(), ws.order_keys.get(), *d_list, n_ptr, n_list, col.n_groups,
                                           c.per_group, stream, st));
    } else {
        FRZ_TRY(frz_launch_collapse(c, *d_list, n_ptr, std::max<uint64_t>(n_list, 1), col.n_groups, capped ? c.per_group : 0, stream, st));
    }
    if (!capped || n_list == 0) return FRZ_OK;
    FrzMatchDev* kept = *d_list == ws.matches_a.get() ? ws.matches_b.get() : ws.matches_a.get();
    FRZ_TRY(retain_rows(m, CollapseKeep{c, *d_list}, *d_list, n_list, kept, stream, st));
    *d_list = kept;
    return FRZ_OK;
}

// The attribute of an ordered call (frz_match_list_ordered): the list is sorted by its order key (order_plan.cuh).
struct Ordering {
    FrzOrderDev dev;   // the attribute, the boost (n_boost == 0: none), the order; `reversed` is set by the call
};

// The ordered call's steps after the list (DESIGN.md §4.15), in place of the sort: the list's length is read back first (a
// survivor-list overflow returns kRetryOverflow there), then the keys are computed and their varying bits read back, and
// the select narrows the list to its first `limit` rows (skipped when they are all of it).  A selection of at most
// kFrzOrderBlockRows rows is sorted by one block, a larger one by the LSD histogram-kernel sort.  *d_list then points at
// the first min(limit, total) rows in order.
frz_status order_list(frz_matcher* m, const FrzCorpusStorage& cs, const Ordering& ord, bool reversed, uint32_t limit,
                      FrzMatchDev** d_list, cudaStream_t stream, FrzLaunchStats* st) {
    FrzWorkspace& ws = m->ws;
    FRZ_TRY(read_counters(m, stream));
    const uint64_t n = ws.h_counters.get()->total;
    if (n <= 1 || limit == 0) return FRZ_OK;   // nothing to order, or nothing to return
    FRZ_TRY(ws.order_keys.reserve(n));
    FRZ_TRY(ws.order_state.reserve(1));
    FRZ_TRY(ws.h_order_state.reserve(1));
    FrzOrderDev o = ord.dev;
    o.reversed = reversed;
    FrzOrderState* dst = ws.order_state.get();
    const unsigned long long* n_ptr = &ws.counters.get()->total;
    FRZ_TRY(frz_launch_order_keys(*d_list, n_ptr, n, o, ws.order_keys.get(), dst, stream, st));
    FRZ_CUDA_TRY(cudaMemcpyAsync(ws.h_order_state.get(), dst, sizeof(FrzOrderState), cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    const FrzOrderState& h = *ws.h_order_state.get();
    uint32_t shifts[kFrzOrderMaxDigits];
    const uint32_t n_shifts = frz_order_digits(h.vary_hi & h.flip_hi, h.vary_lo & h.flip_lo, shifts);
    const uint64_t k = std::min<uint64_t>(limit, n);
    const bool select = k < n;
    // with k rows to return, a block-sorted selection may stop as soon as it fits in the block (frz_order_pick's fit)
    const uint64_t fit = k <= kFrzOrderBlockRows ? kFrzOrderBlockRows : 0;
    const uint64_t n_sel_max = select && !fit ? k : fit ? std::min<uint64_t>(n, fit) : n;
    const unsigned long long* sel_n = n_ptr;
    const uint32_t* sel = nullptr;
    if (select && !(fit && n <= fit)) {
        FRZ_TRY(ws.order_cand.reserve(2 * n));
        FRZ_TRY(ws.order_sel.reserve(n));
        if (!ws.order_hist.get()) {
            FRZ_TRY(ws.order_hist.reserve(kFrzOrderBins));
            FRZ_CUDA_TRY(cudaMemsetAsync(ws.order_hist.get(), 0, kFrzOrderBins * sizeof(uint32_t), stream));
        }
        FRZ_TRY(frz_launch_order_select(ws.order_keys.get(), dst, ws.order_hist.get(), ws.order_cand.get(), ws.order_sel.get(), n, k,
                                        shifts, n_shifts, fit, stream, st));
        sel_n = &dst->n_sel;
        sel = ws.order_sel.get();
    }
    FrzMatchDev* other = *d_list == ws.matches_a.get() ? ws.matches_b.get() : ws.matches_a.get();
    if (n_sel_max <= kFrzOrderBlockRows) {
        FRZ_TRY(frz_launch_order_sort_block(*d_list, ws.order_keys.get(), sel, sel_n, limit, other, stream, st));
        *d_list = other;
        return FRZ_OK;
    }
    FRZ_TRY(ensure_multi_buffers(m, cs.n));
    if (sel) {   // the selection's rows in a list of their own, sorted back into the list's buffer
        FRZ_TRY(frz_launch_order_gather(*d_list, sel, sel_n, k, other, stream, st));
        FRZ_TRY(frz_launch_sort_by_order_dev(other, ws.multi_a.get(), *d_list, sel_n, o, shifts, n_shifts, ws.sort, stream, st, limit));
        return FRZ_OK;
    }
    FRZ_TRY(frz_launch_sort_by_order_dev(*d_list, ws.multi_a.get(), other, n_ptr, o, shifts, n_shifts, ws.sort, stream, st, limit));
    *d_list = other;
    return FRZ_OK;
}

// The sort strategies' two halves: the list's index direction, and whether it is sorted by score.
bool sort_reversed(uint8_t sort) { return sort == FRZ_SORT_INDEX_DESC || sort == FRZ_SORT_SCORE_THEN_INDEX_DESC; }
bool sort_by_score(uint8_t sort) { return sort == FRZ_SORT_SCORE_THEN_INDEX_ASC || sort == FRZ_SORT_SCORE_THEN_INDEX_DESC; }
// What a collapse's order keys rank by: the ranking's key, else the score when the list is sorted by score, else the index.
uint8_t collapse_order(bool ranked, bool by_score) {
    return ranked ? FRZ_COLLAPSE_BY_KEY : by_score ? FRZ_COLLAPSE_BY_SCORE : FRZ_COLLAPSE_BY_INDEX;
}

// What a list call asks for (match_list_device, match_list_host): Matcher::match_list in `sort` order, truncated to its
// first `limit` rows (top-K calls: only those positions of the final list are written, the sort's last scatter and the
// final copy drop the rest; the count in ws.counters->total stays the full match count).  scope: as in match_into_device.
// rank: sort by the ranking's key instead, under every strategy and for the empty matcher too (the strategy's direction
// only orders ties).  col: collapse the list before its sort (collapse_list; with ord, by the order key, so each group
// keeps its first rows in the ordered list); group_counts (host, col->n_groups entries)
// receives the list's rows per group.  cols: the list is that of a frz_match_list_columns call, whose starting column is
// the call's corpus (match_patterns).  ord: order the list by the attribute instead (order_list), under every strategy and
// for the empty matcher too.  col, cols and ord are for host calls only; the shard calls set index_offset and final_out
// (device, >= corpus length: where the final list must land).
struct ListCall {
    uint8_t sort = FRZ_SORT_INDEX_ASC;
    uint64_t limit = UINT64_MAX;
    uint32_t index_offset = 0;
    FrzMatchDev* final_out = nullptr;
    SubsetScope scope;
    std::optional<Ranking> rank;
    std::optional<Collapse> col;
    std::optional<Columns> cols;
    std::optional<Ordering> ord;
    uint32_t* group_counts = nullptr;

    // a list never holds more than 2^32 - 1 matches
    uint32_t dev_limit() const { return (uint32_t)std::min<uint64_t>(limit, kFrzNoLimit); }
    // `!self.patterns.is_empty() && sort.is_by_score()` (src/matcher/mod.rs:218), and every ranked or ordered call
    bool will_sort(const frz_matcher& m) const {
        return rank || ord || (sort_by_score(sort) && (cols ? cols->any_compiled : !m.compiled.empty()));
    }
    // the fused histogram counts the scores of every row of the list, so only a plain score sort may use it
    bool fused_hist(const frz_matcher& m) const { return will_sort(m) && !rank && !col && !ord; }
    // where the scoring kernels may write the list: final_out when no sort follows them
    FrzMatchDev* scoring_out(const frz_matcher& m) const { return will_sort(m) ? nullptr : final_out; }
};

frz_status match_list_device(frz_matcher* m, const FrzCorpusStorage& cs, const ListCall& call, FrzMatchDev** d_result,
                             cudaStream_t stream, FrzLaunchStats* st) {
    FrzWorkspace& ws = m->ws;
    const bool reversed = sort_reversed(call.sort);
    const bool will_sort = call.will_sort(*m);
    const uint32_t limit = call.dev_limit();
    const auto& rank = call.rank;
    FrzMatchDev* const final_out = call.final_out;
    reset_call_state(m);
    FrzMatchDev* d_list = nullptr;
    uint32_t bound = 0;
    FrzScoreHist hist;
    if (call.cols) FRZ_TRY(match_patterns(m, call.cols->pats, cs, call.cols->live, call.index_offset, reversed, &d_list, &bound, stream, st,
                                          call.scope));
    else FRZ_TRY(match_into_device(m, cs, call.index_offset, reversed, &d_list, &bound, stream, st, call.scoring_out(*m),
                                   call.fused_hist(*m) ? &hist : nullptr, call.scope));
    if (call.col)
        FRZ_TRY(collapse_list(m, cs, *call.col, collapse_order(rank.has_value(), will_sort), reversed, rank, call.ord ? &call.ord->dev : nullptr,
                              &d_list, stream, st));
    if (call.ord) {
        FRZ_TRY(order_list(m, cs, *call.ord, reversed, limit, &d_list, stream, st));
    } else if (will_sort) {
        if (rank) bound = (uint32_t)std::min<uint64_t>((uint64_t)bound + rank->max_boost, 0xFFFF);   // the key bound
        FrzMatchDev* other = final_out ? final_out : (d_list == ws.matches_a.get() ? ws.matches_b.get() : ws.matches_a.get());
        // two-pass sort (score bound >= 1024) needs a scratch list of the corpus size: the multi-pattern ping-pong
        // buffer is free at this point (d_list is never multi_a); grow it whenever THIS corpus is larger
        FrzMatchDev* tmp = nullptr;
        if (bound >= 1024) {
            FRZ_TRY(ensure_multi_buffers(m, cs.n));
            tmp = ws.multi_a.get();
        }
        const unsigned long long* n_ptr = &ws.counters.get()->total;
        if (rank) {
            FRZ_TRY(frz_launch_sort_by_key_dev(d_list, tmp, other, n_ptr, rank->boost, rank->n, bound, ws.sort, stream, st, limit));
        } else {
            if (hist.counts) FRZ_TRY(frz_launch_sort_fused(d_list, other, n_ptr, hist, ws.sort, stream, st, limit));
            else FRZ_TRY(frz_launch_sort_by_score_dev(d_list, tmp, other, n_ptr, bound, ws.sort, stream, st, limit));
            m->last_sort_bins = frz_sort_single_pass_bins(bound);   // a per-score table (the multi-GPU merge reads it)
        }
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

// The call (match_list_device) → host: its first min(call.limit, total) rows (copy_out).
frz_status match_list_host(frz_matcher* m, const frz_corpus* corpus, const ListCall& call, frz_match* out, uint64_t cap, uint64_t* n_out,
                           uint64_t* n_total) {
    const auto& col = call.col;
    if (call.scope.none) {
        if (n_out) *n_out = 0;
        if (n_total) *n_total = 0;
        if (col && call.group_counts) memset(call.group_counts, 0, col->n_groups * sizeof(uint32_t));
        return FRZ_OK;
    }
    cudaStream_t stream = nullptr;
    FrzLaunchStats st;
    FrzMatchDev* d_list = nullptr;
    frz_status s = FRZ_OK;
    for (int attempt = 0; attempt < 2; attempt++) {
        s = match_list_device(m, corpus->st, call, &d_list, stream, &st);
        if (s == FRZ_OK) s = copy_out(m, d_list, call.limit, out, cap, n_out, n_total, stream);
        if (s != kRetryOverflow) break;
        FRZ_TRY(ensure_workspace(m, corpus->st, std::max<uint64_t>(corpus->st.n, 1)));  // worst-case lists, then once more
    }
    if (s == kRetryOverflow) s = frz_fail(FRZ_ERR_CUDA, "survivor list overflow persisted");
    if (s == FRZ_OK && col && call.group_counts) {
        FRZ_CUDA_TRY(cudaMemcpyAsync(call.group_counts, m->ws.collapse_counts.get(), col->n_groups * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                                     stream));
        FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    }
    collect_timings(m, st);
    return s;
}

}  // namespace

// ---------------------------------------------------------------------------------- batched top-K
// frz_match_list_batch_ordered, frz_match_list_batch_collapsed, frz_match_list_batch and frz_match_list_batch_top
// (DESIGN.md §4.11), and frz_match_list_batch_columns (§4.13).  Queries of the batched class run in sub-batches whose
// every stage is one launch (per kernel variant present, and per column) over all of the sub-batch's queries, with one
// upload, one read-back and one synchronise per sub-batch; ordered queries run in sub-batches of their own.  Every other
// query, and every query of an overflowed sub-batch, runs its single-query call's pipeline (frz_match_list_top,
// _subset_top, _ranked, _collapsed, _ordered, _ordered_collapsed or _columns).  The entry points follow the column calls.
namespace {

// Device scratch of one sub-batch's queries, in one allocation: a fixed budget, so a batch call holds the same scratch for
// every q (its size depends on the corpus: larger corpora get smaller sub-batches, and a corpus whose queries do not fit two
// to a sub-batch is answered query by query).  A call with grouped queries adds each query's group tables at the largest
// n_groups among its batched grouped queries (batch_collapse_plan.cuh), so its sub-batches hold fewer queries; a grouped
// query whose tables alone do not fit two to a sub-batch (more than about 22 M groups) runs frz_match_list_collapsed.
constexpr uint64_t kBatchScratchBytes = 512ull << 20;
// Where the batched path is faster than a loop of frz_match_list_top (tools/bench_batch.py on an H100 SXM, DESIGN.md §4.11):
// at 100 k rows from 64 queries on, not at 8 queries (the call's fixed costs); at 1 M rows for max_typos = 0 queries only
// (with a typo budget, short needles pass more rows than the survivor lists hold, and the overflowed sub-batches run
// again query by query).  Elsewhere the call runs the loop.
constexpr uint64_t kBatchMaxRows = 1ull << 18;
constexpr uint64_t kBatchMaxRowsNoTypo = 1ull << 21;   // FRZ_T_0 queries
constexpr uint64_t kBatchMinQueries = 32;
// A grouped query that wants the counts of more groups than this runs frz_match_list_collapsed: its counts' read-back
// through the sub-batch's staging then costs more than the loop saves (tools/bench_batch_collapsed.py on an H100 SXM,
// DESIGN.md §4.11: ahead of the loop with 100 k groups, behind it with 1 M).
constexpr uint64_t kBatchMaxCountedGroups = 1ull << 18;
// A column query (frz_match_list_batch_columns) with a typo budget in some column batches only up to this many rows, and
// one whose every pattern has max_typos = 0 only up to kBatchMaxRows (tools/bench_batch_columns.py on an H100 SXM, DESIGN.md
// §4.13: with a typo budget, or at 1 M rows, the short needles of a second column pass more rows than the survivor lists
// hold, and the overflowed sub-batches run again query by query, behind the loop).
constexpr uint64_t kBatchColumnsMaxRowsTypo = 0;
// The limits in force (frz_debug_batch_limits changes them for tests and tools/bench_batch.py) and what the calling
// thread's last batch call did (frz_debug_batch_last).
std::atomic<uint64_t> g_batch_max_rows{kBatchMaxRows};
std::atomic<uint64_t> g_batch_columns_typo_rows{kBatchColumnsMaxRowsTypo};
std::atomic<uint64_t> g_batch_min_queries{kBatchMinQueries};
thread_local uint64_t g_batch_last[4] = {0, 0, 0, 0};   // batched queries, overflowed queries, sub-batches, launches

struct BatchLayout {
    uint64_t nt = 0, stride = 0, cap = 0, k = 0;
    uint64_t groups = 0;     // entries of each query slot's group tables (0: no query of the call has groups)
    uint64_t n_cols = 0;     // columns of a frz_match_list_batch_columns call (0: a single-corpus call)
    bool ordered = false;    // the call has batched ordered queries (batch_order_plan.cuh's arrays)
    uint64_t off[28] = {};   // byte offsets of the arrays below, in this order
    uint64_t bytes = 0;
    enum { CTR, BITMAP, PREFIX, TCOUNT, TBASE, SURV, LISTS, BEST, TAKEN, ACC, JERR, PATS, REV, BYSC, SCOPE, COLS, CMAP, ORD, TOTALS, ROWS,
           COUNTS, KEYS, CAND, SEL, STATE, HIST, BESTLO, END };
    // queries per sub-batch for this corpus and k (0: fewer than two fit the budget)
    static uint64_t per_query(const FrzCorpusStorage& cs, uint64_t k, uint64_t cap) {
        const uint64_t nt = cs.n_tiles;
        return sizeof(FrzCounters) + nt * 32 * (sizeof(uint32_t) + sizeof(uint16_t)) + nt * (sizeof(uint32_t) + sizeof(uint64_t)) +
               FRZ_N_CLASSES * cap * sizeof(FrzSurvivor) + std::max<uint64_t>(cs.n, 1) * sizeof(FrzMatchDev) + sizeof(FrzPatternDev) + 2 +
               sizeof(FrzBatchScope) + sizeof(unsigned long long) + k * sizeof(FrzMatchDev) + 13 * 256 / 2;
    }
    // n_cols_ > 0 (a column call) adds each query's accumulator and error word, a pattern slot per column and query, and
    // the fold records (batch_columns_plan.cuh); a single-corpus call gets the layout it had before column calls existed.
    // ordered_ adds the ordered sub-batches' arrays (ORD is uploaded with the patterns; the rest follow the read-back and
    // take no room, not even alignment, without ordered queries: such a call gets the layout it had before them)
    BatchLayout(const FrzCorpusStorage& cs, uint64_t k_, uint64_t cap_, uint64_t qs, uint64_t groups_ = 0, uint64_t n_cols_ = 0,
                bool ordered_ = false)
        : nt(cs.n_tiles), stride(std::max<uint64_t>(cs.n, 1)), cap(cap_), k(k_), groups(groups_), n_cols(n_cols_), ordered(ordered_) {
        const uint64_t g = groups ? qs : 0;   // the group arrays exist only in a call with grouped queries
        const uint64_t c = n_cols ? qs : 0;   // the join arrays only in a column call
        const uint64_t o = ordered ? qs : 0;  // the ordering arrays only in a call with ordered queries
        const uint64_t size[END] = {qs * sizeof(FrzCounters), qs * nt * 32 * sizeof(uint32_t), qs * nt * 32 * sizeof(uint16_t),
                                    qs * nt * sizeof(uint32_t), qs * nt * sizeof(uint64_t), qs * FRZ_N_CLASSES * cap * sizeof(FrzSurvivor),
                                    qs * stride * sizeof(FrzMatchDev), g * groups * sizeof(unsigned long long), g * stride,
                                    c * stride * sizeof(uint32_t), c * sizeof(uint32_t),
                                    qs * std::max<uint64_t>(n_cols, 1) * sizeof(FrzPatternDev), qs, qs, qs * sizeof(FrzBatchScope),
                                    g * sizeof(FrzBatchCollapse), c * (n_cols * sizeof(FrzColumnFold) + 1), o * sizeof(FrzOrderDev),
                                    qs * sizeof(unsigned long long), qs * k * sizeof(FrzMatchDev), g * groups * sizeof(uint32_t),
                                    o * stride * sizeof(FrzOrderKey), o * 2 * stride * sizeof(uint32_t), o * kFrzOrderBlockRows * sizeof(uint32_t),
                                    o * sizeof(FrzOrderState), o * kFrzOrderBins * sizeof(uint32_t), (g && o) * g * groups * sizeof(unsigned long long)};
        uint64_t at = 0;
        for (int i = 0; i < END; i++) {
            // CTR..BITMAP are zeroed as one range, ACC..JERR too, PATS..ORD uploaded as one, TOTALS..COUNTS read back as one,
            // STATE..HIST zeroed as one
            const bool packed = i == BITMAP || i == JERR || i == REV || i == BYSC || i == SCOPE || i == COLS || i == CMAP || i == ORD ||
                                i == ROWS || i == COUNTS || i == HIST;
            if (i > COUNTS && !size[i]) {
                off[i] = at;
                continue;
            }
            if (!packed) at = (at + 255) & ~255ull;
            else at = (at + 7) & ~7ull;
            off[i] = at;
            at += size[i];
        }
        off[END] = at;
        bytes = at;
    }
};

// the survivor-list length per class and query: frz_match_list_top's first attempt (initial_survivor_cap, which is the
// same for every pattern that is not FRZ_T_NONE)
uint64_t batch_survivor_cap(const FrzCorpusStorage& cs) {
    return std::min<uint64_t>(std::max<uint64_t>(cs.n / 4, 1 << 16), std::max<uint64_t>(cs.n, 1));
}

// the batched class: one compiled fuzzy byte pattern of up to FRZ_MAX_NEEDLE bytes, not negated (and, when it can match
// every row, a survivor list that can hold them all)
bool batchable(const frz_matcher* m, const FrzCorpusStorage& cs) {
    if (m->compiled.size() != 1) return false;
    const Compiled& c = m->compiled[0];
    if (c.negated || c.literal || c.unicode || c.is_long() || c.dev.typo_mode == FRZ_T_LITERAL) return false;
    return c.dev.typo_mode != FRZ_T_NONE || batch_survivor_cap(cs) >= std::max<uint64_t>(cs.n, 1);
}
// the selection of the batched path for such a query (kBatchMaxRows, kBatchMaxRowsNoTypo)
bool batch_selected(const frz_matcher* m, const FrzCorpusStorage& cs) {
    const uint64_t max_rows = g_batch_max_rows.load();
    const uint64_t limit = m->compiled[0].dev.typo_mode == FRZ_T_0 ? std::max(max_rows, kBatchMaxRowsNoTypo) : max_rows;
    return cs.n <= limit;
}

// The columns of a frz_match_list_batch_columns call: query j's matcher for column c is ms[j * n_cols + c].
struct BatchColumns {
    const frz_corpus* const* cols = nullptr;
    uint64_t n_cols = 0;
    uint8_t sort = 0;
};
// the batched class of a column query: every column's matcher of the batched class or without a pattern, at least one
// pattern, at most kFrzBatchMaxColumns columns, and rows within the row limit (g_batch_max_rows when every pattern has
// max_typos = 0, else g_batch_columns_typo_rows)
bool batch_columns_selected(frz_matcher* const* mj, const BatchColumns& bc) {
    if (bc.n_cols > kFrzBatchMaxColumns) return false;
    bool any = false, all_t0 = true;
    for (uint64_t c = 0; c < bc.n_cols; c++) {
        const frz_matcher* m = mj[c];
        if (m->compiled.empty()) continue;
        if (!batchable(m, bc.cols[c]->st)) return false;
        any = true;
        all_t0 &= m->compiled[0].dev.typo_mode == FRZ_T_0;
    }
    return any && bc.cols[0]->st.n <= (all_t0 ? g_batch_max_rows.load() : g_batch_columns_typo_rows.load());
}

// The groups of a call's queries, indexed as ms (frz_match_list_batch_collapsed).
struct BatchGroups {
    const FrzBatchCollapse* cols = nullptr;   // [j] ids == nullptr: no groups (cols == nullptr: no query of the call has any)
    const uint64_t* n_groups = nullptr;       // [j]
    uint32_t* const* counts = nullptr;        // [j] the caller's count array, or nullptr (counts == nullptr: none)
};

// One sub-batch: queries which[0..ns) of ms, all of the batched class.  scopes: nullptr when no query of the call is scoped
// or ranked, else every query's subset and boost (indexed as ms).  gr: the call's groups (L.groups > 0 when it has any).
// bc: a column call (c is its column 0): each column's stages run for the queries with a pattern in it, in slots of their
// own, and the join (batch_columns.cu) leaves each query's list where the cut reads it.
// ords: an ordered sub-batch (frz_match_list_batch_ordered, L.ordered), every query's attribute, boost and order (indexed
// as ms); its last stage orders each query's rows by its order key (order.cu) in place of the cut.
// *overflow: a survivor list overflowed, nothing was written to the results (the caller runs the queries one by one).
frz_status batch_run(frz_matcher* const* ms, const FrzBatchScope* scopes, const BatchGroups& gr, const uint64_t* which, uint32_t ns,
                     const frz_corpus* c, uint64_t k, const BatchLayout& L, uint8_t* d, frz_match* out, uint64_t* n_out,
                     uint64_t* n_total, bool* overflow, FrzLaunchStats& st, const BatchColumns* bc = nullptr,
                     const FrzOrderDev* ords = nullptr) {
    const FrzCorpusStorage& cs = c->st;
    cudaStream_t stream = nullptr;
    *overflow = false;
    const uint64_t up = L.off[BatchLayout::TOTALS] - L.off[BatchLayout::PATS];
    FRZ_TRY(c->batch_stage.reserve(std::max(up, L.off[BatchLayout::KEYS] - L.off[BatchLayout::TOTALS])));
    uint8_t* h = c->batch_stage.get();
    FrzPatternDev* h_pats = reinterpret_cast<FrzPatternDev*>(h);
    uint8_t* h_rev = h + (L.off[BatchLayout::REV] - L.off[BatchLayout::PATS]);
    uint8_t* h_bysc = h + (L.off[BatchLayout::BYSC] - L.off[BatchLayout::PATS]);
    FrzBatchScope* h_scope = reinterpret_cast<FrzBatchScope*>(h + (L.off[BatchLayout::SCOPE] - L.off[BatchLayout::PATS]));
    FrzBatchCollapse* h_cols = reinterpret_cast<FrzBatchCollapse*>(h + (L.off[BatchLayout::COLS] - L.off[BatchLayout::PATS]));
    bool scoped = false;   // a query of the sub-batch is scoped or ranked: the last stage is k_batch_top<ScopedKey>
    uint8_t grouped[kFrzBatchMaxSub] = {}, wants[kFrzBatchMaxSub] = {};
    uint32_t slot[kFrzBatchMaxSub] = {}, n_grouped = 0, rounds = 0;
    for (uint32_t j = 0; j < ns; j++) {
        const uint8_t sort = bc ? bc->sort : ms[which[j]]->config.sort;
        if (!bc) h_pats[j] = ms[which[j]]->compiled[0].dev;
        h_rev[j] = sort_reversed(sort);
        h_bysc[j] = sort_by_score(sort);
        h_scope[j] = scopes ? scopes[which[j]] : FrzBatchScope();
        scoped |= h_scope[j].scoped || h_scope[j].ranked;
        if (gr.cols && gr.cols[which[j]].ids) {
            grouped[j] = 1;
            wants[j] = gr.counts && gr.counts[which[j]];
            n_grouped++;
            rounds = std::max(rounds, frz_batch_collapse_rounds(gr.cols[which[j]].per_group));
        }
    }
    // the group tables: a slot per grouped query, those whose counts are read back first
    const uint32_t n_back = frz_batch_collapse_slots(grouped, wants, ns, slot);
    for (uint32_t j = 0; j < ns && L.groups; j++) {
        h_cols[j] = gr.cols[which[j]];
        h_cols[j].table = frz_batch_collapse_table(slot[j], L.groups);
    }
    // a column call's patterns: column c's queries with a pattern take its slots 0, 1, ... in query order
    FrzColumnFold* h_fold = reinterpret_cast<FrzColumnFold*>(h + (L.off[BatchLayout::CMAP] - L.off[BatchLayout::PATS]));
    uint8_t* h_need = reinterpret_cast<uint8_t*>(h_fold + L.n_cols * ns);
    std::vector<uint32_t> n_slots(L.n_cols, 0);
    std::vector<uint8_t> folded(L.n_cols, 0);
    for (uint32_t j = 0; j < ns && bc; j++) h_need[j] = 0;
    for (uint64_t col = 0; col < L.n_cols; col++) {
        for (uint32_t j = 0; j < ns; j++) {
            const frz_matcher* m = ms[which[j] * L.n_cols + col];
            FrzColumnFold& f = h_fold[col * ns + j];
            f.pass = h_need[j];
            if (!m->compiled.empty()) {
                f.slot = (uint8_t)n_slots[col];
                h_pats[col * ns + n_slots[col]++] = m->compiled[0].dev;
            } else {
                f.slot = bc->cols[col]->st.n_removed ? kFrzColumnLive : kFrzColumnSkip;
            }
            if (f.slot != kFrzColumnSkip) { h_need[j]++; folded[col] = 1; }
        }
    }
    // an ordered sub-batch's attributes, with each query's list direction
    FrzOrderDev* h_ord = reinterpret_cast<FrzOrderDev*>(h + (L.off[BatchLayout::ORD] - L.off[BatchLayout::PATS]));
    for (uint32_t j = 0; j < ns && ords; j++) {
        h_ord[j] = ords[which[j]];
        h_ord[j].reversed = h_rev[j];
    }
    const uint64_t down = L.off[BatchLayout::COUNTS] + n_back * L.groups * sizeof(uint32_t) - L.off[BatchLayout::TOTALS];
    FrzBatchDev b;
    b.pats = reinterpret_cast<const FrzPatternDev*>(d + L.off[BatchLayout::PATS]);
    b.reversed = d + L.off[BatchLayout::REV];
    b.by_score = d + L.off[BatchLayout::BYSC];
    b.surv = reinterpret_cast<FrzSurvivor*>(d + L.off[BatchLayout::SURV]);
    b.surv_cap = L.cap;
    b.ctr = reinterpret_cast<FrzCounters*>(d + L.off[BatchLayout::CTR]);
    b.surv_bitmap = reinterpret_cast<uint32_t*>(d + L.off[BatchLayout::BITMAP]);
    b.word_prefix = reinterpret_cast<uint16_t*>(d + L.off[BatchLayout::PREFIX]);
    b.tile_count = reinterpret_cast<uint32_t*>(d + L.off[BatchLayout::TCOUNT]);
    b.tile_out_base = reinterpret_cast<uint64_t*>(d + L.off[BatchLayout::TBASE]);
    b.lists = reinterpret_cast<FrzMatchDev*>(d + L.off[BatchLayout::LISTS]);
    b.list_stride = L.stride;
    unsigned long long* totals = reinterpret_cast<unsigned long long*>(d + L.off[BatchLayout::TOTALS]);
    FrzMatchDev* rows = reinterpret_cast<FrzMatchDev*>(d + L.off[BatchLayout::ROWS]);
    FRZ_CUDA_TRY(cudaMemcpyAsync(d + L.off[BatchLayout::PATS], h, up, cudaMemcpyHostToDevice, stream));
    // the counters and survivor bitmaps of the first nq slots start zero
    const auto clear_slots = [&](uint32_t nq) {
        return cudaMemsetAsync(d + L.off[BatchLayout::CTR], 0,
                               L.off[BatchLayout::BITMAP] + (uint64_t)nq * L.nt * 32 * sizeof(uint32_t) - L.off[BatchLayout::CTR], stream);
    };
    if (!bc) {
        FRZ_CUDA_TRY(clear_slots(ns));
        const FrzCorpusView cv = cs.view();
        FRZ_TRY(frz_launch_prefilter_batch(cv, b, h_pats, ns, stream, &st));
        FRZ_TRY(frz_launch_sw_batch(cv, b, h_pats, ns, stream, &st));
    } else {   // each column's stages, folded into the accumulators, then every query's joined list
        FrzBatchColumnsDev jd;
        jd.acc = reinterpret_cast<uint32_t*>(d + L.off[BatchLayout::ACC]);
        jd.err = reinterpret_cast<uint32_t*>(d + L.off[BatchLayout::JERR]);
        jd.fold = reinterpret_cast<const FrzColumnFold*>(d + L.off[BatchLayout::CMAP]);
        jd.need = d + L.off[BatchLayout::CMAP] + (h_need - reinterpret_cast<uint8_t*>(h_fold));
        jd.n_rows = cs.n;
        FRZ_CUDA_TRY(cudaMemsetAsync(jd.acc, 0, L.off[BatchLayout::JERR] + ns * sizeof(uint32_t) - L.off[BatchLayout::ACC], stream));
        for (uint64_t col = 0; col < L.n_cols; col++) {
            const FrzCorpusView cv = bc->cols[col]->st.view();
            FrzBatchDev bcol = b;
            bcol.pats = b.pats + col * ns;
            if (n_slots[col]) {
                FRZ_CUDA_TRY(clear_slots(n_slots[col]));
                FRZ_TRY(frz_launch_prefilter_batch(cv, bcol, h_pats + col * ns, n_slots[col], stream, &st));
                FRZ_TRY(frz_launch_sw_batch(cv, bcol, h_pats + col * ns, n_slots[col], stream, &st));
            }
            if (folded[col]) FRZ_TRY(frz_launch_batch_columns_fold(bcol, jd, cv, (uint32_t)col, ns, stream, &st));
        }
        FRZ_TRY(frz_launch_batch_columns_join(b, jd, (uint32_t)L.nt, ns, stream, &st));
    }
    const FrzBatchScope* d_scope = reinterpret_cast<const FrzBatchScope*>(d + L.off[BatchLayout::SCOPE]);
    FrzBatchTables t = {};
    t.scopes = d_scope;
    if (L.groups) {
        t.cols = reinterpret_cast<const FrzBatchCollapse*>(d + L.off[BatchLayout::COLS]);
        t.counts = reinterpret_cast<uint32_t*>(d + L.off[BatchLayout::COUNTS]);
        t.best = reinterpret_cast<unsigned long long*>(d + L.off[BatchLayout::BEST]);
        t.taken = d + L.off[BatchLayout::TAKEN];
    }
    if (ords) {   // the keys, the collapse on them, then each query's rows selected and sorted by key
        FrzBatchOrderDev od;
        od.ords = reinterpret_cast<const FrzOrderDev*>(d + L.off[BatchLayout::ORD]);
        od.keys = reinterpret_cast<FrzOrderKey*>(d + L.off[BatchLayout::KEYS]);
        od.cand = reinterpret_cast<uint32_t*>(d + L.off[BatchLayout::CAND]);
        od.sel = reinterpret_cast<uint32_t*>(d + L.off[BatchLayout::SEL]);
        od.st = reinterpret_cast<FrzOrderState*>(d + L.off[BatchLayout::STATE]);
        od.hist = reinterpret_cast<uint32_t*>(d + L.off[BatchLayout::HIST]);
        od.best_lo = reinterpret_cast<unsigned long long*>(d + L.off[BatchLayout::BESTLO]);
        FRZ_CUDA_TRY(cudaMemsetAsync(od.st, 0, L.off[BatchLayout::HIST] + (uint64_t)ns * kFrzOrderBins * sizeof(uint32_t) - L.off[BatchLayout::STATE],
                                     stream));
        FRZ_TRY(frz_launch_batch_order_keys(b, od, ns, stream, &st));
        if (n_grouped) {
            FRZ_CUDA_TRY(cudaMemsetAsync(t.counts, 0, n_grouped * L.groups * sizeof(uint32_t), stream));
            FRZ_TRY(frz_launch_batch_collapse_by_key(b, t, od, ns, rounds, stream, &st));
        }
        FRZ_TRY(frz_launch_batch_order_top(b, t, od, ns, (uint32_t)k, rows, totals, stream, &st));
    } else if (n_grouped) {   // the collapse, then the kept rows' cut
        FRZ_CUDA_TRY(cudaMemsetAsync(t.counts, 0, n_grouped * L.groups * sizeof(uint32_t), stream));
        FRZ_TRY(frz_launch_batch_collapse(b, t, ns, rounds, stream, &st));
        FRZ_TRY(frz_launch_batch_top_collapsed(b, t, ns, (uint32_t)k, rows, totals, stream, &st));
    } else {
        FRZ_TRY(frz_launch_batch_top(b, scoped ? d_scope : nullptr, ns, (uint32_t)k, rows, totals, stream, &st));
    }
    // the staged patterns are not read again: the read-back may reuse the staging
    FRZ_CUDA_TRY(cudaMemcpyAsync(h, totals, down, cudaMemcpyDeviceToHost, stream));
    FRZ_CUDA_TRY(cudaStreamSynchronize(stream));
    const unsigned long long* h_totals = reinterpret_cast<const unsigned long long*>(h);
    const frz_match* h_rows = reinterpret_cast<const frz_match*>(h + (L.off[BatchLayout::ROWS] - L.off[BatchLayout::TOTALS]));
    const uint32_t* h_counts = reinterpret_cast<const uint32_t*>(h + (L.off[BatchLayout::COUNTS] - L.off[BatchLayout::TOTALS]));
    for (uint32_t j = 0; j < ns; j++)
        if (h_totals[j] == kFrzBatchOverflow) { *overflow = true; return FRZ_OK; }
    for (uint32_t j = 0; j < ns; j++) {
        const uint64_t q = which[j], n = frz_batch_rows(k, h_totals[j]);
        n_out[q] = n;
        if (n_total) n_total[q] = h_totals[j];
        if (n) memcpy(out + q * k, h_rows + frz_batch_row0(j, k), n * sizeof(frz_match));
        if (wants[j]) memcpy(gr.counts[q], h_counts + frz_batch_collapse_table(slot[j], L.groups), gr.n_groups[q] * sizeof(uint32_t));
    }
    return FRZ_OK;
}

}  // namespace

extern "C" void frz_debug_batch_limits(uint64_t max_rows, uint64_t min_queries) {
    g_batch_max_rows = max_rows ? max_rows : kBatchMaxRows;
    g_batch_columns_typo_rows = max_rows ? max_rows : kBatchColumnsMaxRowsTypo;
    g_batch_min_queries = min_queries ? min_queries : kBatchMinQueries;
}

extern "C" void frz_debug_batch_last(uint64_t out[4]) {
    for (int i = 0; i < 4; i++) out[i] = g_batch_last[i];
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
    // frz_subset_where's grow-only scratch
    FrzDevArray<uint32_t> chunk_count;      // members per chunk of kFrzWhereChunk indices
    FrzDevArray<uint64_t> chunk_base;       // their exclusive scan
    FrzDevArray<FrzCounters> counters;      // ->total: the member count k_scan_blocks leaves
    FrzDevArray<int64_t> sets;              // every set clause's sorted distinct values
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

// ---------------------------------------------------------------------------------- per-row handles
static_assert(kFrzAttrNull == FRZ_ATTR_NULL && kFrzWhereMaxClauses == FRZ_WHERE_MAX_CLAUSES && kFrzWhereMaxIn == FRZ_WHERE_MAX_IN,
              "where_plan.cuh mirrors frz_cuda.h");

// A value per index of one corpus, on its device, kept by index across corpus edits.  Indices at and past `values.cap()`
// hold kFill.  The corpus comes first: the argument checks and frz_subset_where read it through any handle.
template <typename T, T kFill>
struct RowValues {
    const frz_corpus* corpus = nullptr;
    FrzDevArray<T> values;
};

// A signed 16-bit boost per index (ranked calls); 0 past the values.
struct frz_boost : RowValues<int16_t, 0> {
    int32_t max_set = 0;   // the largest value ever set, at least 0: bounds every boost (the sort's key bound)
};
// A group id per index (collapsed calls); in no group past the values.
struct frz_groups : RowValues<uint32_t, FRZ_GROUP_NONE> {
    uint64_t n_groups = 0;
};
// A signed 64-bit value per index (frz_subset_where, ordered calls); null past the values.
struct frz_attr : RowValues<int64_t, kFrzAttrNull> {};

namespace {
template <typename T>
struct RowSet {   // one (index, value) pair of a *_set call
    uint32_t index;
    T value;
};

template <typename T>
__global__ void k_row_values_scatter(const RowSet<T>* __restrict__ set, uint64_t n, T* __restrict__ values) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (uint64_t)gridDim.x * blockDim.x)
        values[set[j].index] = set[j].value;
}

template <typename T>
__global__ void k_row_values_fill(T* __restrict__ values, uint64_t from, uint64_t to, T fill) {
    for (uint64_t i = from + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < to; i += (uint64_t)gridDim.x * blockDim.x)
        values[i] = fill;
}

frz_status no_check() { return FRZ_OK; }

// frz_*_create: a handle of c holding values[0, n).  what: the values' name in the length message; check: the handle's
// own checks, after the length.
template <class H, typename T, class Check>
frz_status row_values_create(const frz_corpus* c, const T* values, uint64_t n, H** out, const char* what, Check check) {
    if (!c || !out || (n && !values)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (n > c->st.n)
        return frz_fail(FRZ_ERR_INVALID_ARG, "%llu %s for a corpus of %llu haystacks", (unsigned long long)n, what, (unsigned long long)c->st.n);
    FRZ_TRY(check());
    auto h = std::make_unique<H>();
    h->corpus = c;
    if (n) {
        FRZ_TRY(frz_ensure_device(c->st.device));
        FRZ_TRY(h->values.reserve(n));
        FRZ_CUDA_TRY(cudaMemcpy(h->values.get(), values, n * sizeof(T), cudaMemcpyHostToDevice));
    }
    *out = h.release();
    return FRZ_OK;
}

// frz_*_set: values[which[j]] = v[j] for rows below the corpus's length, each at most once.  check: the handle's own checks
// on v, before the duplicate check.  An index past the values first grows them to the corpus's length, the old values kept
// and the new ones kFill (FrzDevArray drops its contents when it grows).
template <typename T, T kFill, class Check>
frz_status row_values_set(RowValues<T, kFill>* h, const uint32_t* which, const T* v, uint64_t n, Check check) {
    if (!h || (n && (!which || !v))) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (n == 0) return FRZ_OK;
    FRZ_TRY(check_indices(h->corpus, which, n));
    FRZ_TRY(check());
    std::vector<uint32_t> sorted(which, which + n);
    std::sort(sorted.begin(), sorted.end());
    for (uint64_t j = 1; j < n; j++)
        if (sorted[j] == sorted[j - 1]) return frz_fail(FRZ_ERR_INVALID_ARG, "index %u is set twice", sorted[j]);
    std::vector<RowSet<T>> set(n);
    for (uint64_t j = 0; j < n; j++) set[j] = RowSet<T>{which[j], v[j]};
    FRZ_TRY(frz_ensure_device(h->corpus->st.device));
    if (sorted.back() >= h->values.cap()) {
        const uint64_t old = h->values.cap(), rows = h->corpus->st.n;
        FrzDevArray<T> grown;
        FRZ_TRY(grown.reserve(rows));
        k_row_values_fill<<<grid_for(rows - old, 256), 256>>>(grown.get(), old, rows, kFill);
        FRZ_CUDA_TRY(cudaGetLastError());
        if (old) FRZ_CUDA_TRY(cudaMemcpy(grown.get(), h->values.get(), old * sizeof(T), cudaMemcpyDeviceToDevice));
        FRZ_CUDA_TRY(cudaStreamSynchronize(nullptr));
        h->values = std::move(grown);
    }
    FrzDevArray<RowSet<T>> d_set;   // one copy, one scatter
    FRZ_TRY(d_set.reserve(n));
    FRZ_CUDA_TRY(cudaMemcpy(d_set.get(), set.data(), n * sizeof(RowSet<T>), cudaMemcpyHostToDevice));
    k_row_values_scatter<<<grid_for(n, 256), 256>>>(d_set.get(), n, h->values.get());
    FRZ_CUDA_TRY(cudaGetLastError());
    FRZ_CUDA_TRY(cudaStreamSynchronize(nullptr));
    return FRZ_OK;
}

// every id is below n_groups or FRZ_GROUP_NONE
frz_status check_group_ids(const uint32_t* ids, uint64_t n, uint64_t n_groups) {
    for (uint64_t j = 0; j < n; j++)
        if (ids[j] != FRZ_GROUP_NONE && ids[j] >= n_groups)
            return frz_fail(FRZ_ERR_INVALID_ARG, "group id %u is not below n_groups = %llu", ids[j], (unsigned long long)n_groups);
    return FRZ_OK;
}
}  // namespace

extern "C" frz_status frz_boost_create(const frz_corpus* c, const int16_t* values, uint64_t n, frz_boost** out) {
    FRZ_TRY(row_values_create(c, values, n, out, "boost values", no_check));
    if (n) (*out)->max_set = std::max<int32_t>(0, *std::max_element(values, values + n));
    return FRZ_OK;
}

extern "C" frz_status frz_boost_set(frz_boost* b, const uint32_t* which, const int16_t* values, uint64_t n) {
    FRZ_TRY(row_values_set(b, which, values, n, no_check));
    if (n) b->max_set = std::max<int32_t>(b->max_set, *std::max_element(values, values + n));
    return FRZ_OK;
}

extern "C" void frz_boost_destroy(frz_boost* b) { delete b; }

extern "C" frz_status frz_groups_create(const frz_corpus* c, const uint32_t* ids, uint64_t n, uint64_t n_groups, frz_groups** out) {
    FRZ_TRY(row_values_create(c, ids, n, out, "group ids", [&]() -> frz_status {
        if (n_groups == 0 || n_groups > FRZ_GROUP_NONE)
            return frz_fail(FRZ_ERR_INVALID_ARG, "n_groups = %llu is not in 1 .. 2^32 - 1", (unsigned long long)n_groups);
        return check_group_ids(ids, n, n_groups);
    }));
    (*out)->n_groups = n_groups;
    return FRZ_OK;
}

extern "C" frz_status frz_groups_set(frz_groups* g, const uint32_t* which, const uint32_t* ids, uint64_t n) {
    return row_values_set(g, which, ids, n, [&] { return check_group_ids(ids, n, g->n_groups); });
}

extern "C" uint64_t frz_groups_count(const frz_groups* g) { return g ? g->n_groups : 0; }
extern "C" void frz_groups_destroy(frz_groups* g) { delete g; }

extern "C" frz_status frz_attr_create(const frz_corpus* c, const int64_t* values, uint64_t n, frz_attr** out) {
    return row_values_create(c, values, n, out, "attribute values", no_check);
}

extern "C" frz_status frz_attr_set(frz_attr* a, const uint32_t* which, const int64_t* values, uint64_t n) {
    return row_values_set(a, which, values, n, no_check);
}

extern "C" void frz_attr_destroy(frz_attr* a) { delete a; }

// ---------------------------------------------------------------------------------- subsets from attributes
namespace {
// The device work of frz_subset_where once every argument has passed: k_where writes the bitmap and the chunk counts,
// k_scan_blocks scans the counts, one 8-byte read-back gives the member count, and k_where_members writes the list.  The
// bitmap is written in place unless it must grow; then into a new array, because `base` may be s's old bitmap.
frz_status where_fill(frz_subset* s, FrzWhereDev& w, const std::vector<int64_t>& sets, const frz_subset* base) {
    const uint64_t n = s->corpus->st.n;
    w.has_base = base != nullptr;   // (read before s is emptied: base may be s)
    w.base = base ? base->bits.get() : nullptr;
    w.n_base = base ? base->n_bits : 0;
    s->n_bits = 0;   // empty until the fill completes
    s->n_members = 0;
    if (n == 0) return FRZ_OK;
    const uint64_t n_words = (n + 31) / 32, n_chunks = (n + kFrzWhereChunk - 1) / kFrzWhereChunk;
    FRZ_TRY(s->chunk_count.reserve(n_chunks));
    FRZ_TRY(s->chunk_base.reserve(n_chunks));
    FRZ_TRY(s->counters.reserve(1));
    if (!sets.empty()) {
        FRZ_TRY(s->sets.reserve(sets.size(), std::max<uint64_t>(sets.size(), 64)));
        FRZ_CUDA_TRY(cudaMemcpy(s->sets.get(), sets.data(), sets.size() * sizeof(int64_t), cudaMemcpyHostToDevice));
    }
    FrzDevArray<uint32_t> grown;
    if (s->bits.cap() < n_words) FRZ_TRY(grown.reserve(n_words));
    w.sets = s->sets.get();
    w.n_sets = (uint32_t)sets.size();
    w.bits = grown.get() ? grown.get() : s->bits.get();
    w.chunk_count = s->chunk_count.get();
    w.n = n;
    FRZ_TRY(frz_launch_where(w, nullptr));
    k_scan_blocks<<<1, 1024>>>(s->chunk_count.get(), s->chunk_base.get(), (uint32_t)n_chunks, s->counters.get());
    FRZ_CUDA_TRY(cudaGetLastError());
    uint64_t total = 0;
    FRZ_CUDA_TRY(cudaMemcpy(&total, &s->counters.get()->total, sizeof(total), cudaMemcpyDeviceToHost));
    if (grown.get()) s->bits = std::move(grown);
    if (total) {
        FRZ_TRY(s->members.reserve(total));
        FRZ_TRY(frz_launch_where_members(s->bits.get(), n, s->chunk_base.get(), s->members.get(), nullptr));
        FRZ_CUDA_TRY(cudaStreamSynchronize(nullptr));
    }
    s->n_bits = n;
    s->n_members = total;
    return FRZ_OK;
}
}  // namespace

extern "C" frz_status frz_subset_where(frz_subset* s, const frz_where_clause* clauses, uint64_t n_clauses, const frz_subset* base) {
    if (!s || (n_clauses && !clauses)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (n_clauses > FRZ_WHERE_MAX_CLAUSES)
        return frz_fail(FRZ_ERR_UNSUPPORTED, "%llu clauses (at most %d)", (unsigned long long)n_clauses, FRZ_WHERE_MAX_CLAUSES);
    uint64_t n_in = 0;
    for (uint64_t j = 0; j < n_clauses; j++) {
        if (!clauses[j].attr || (clauses[j].n_in && !clauses[j].in)) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument in clause %llu", (unsigned long long)j);
        n_in += std::min<uint64_t>(clauses[j].n_in, (uint64_t)FRZ_WHERE_MAX_IN + 1);   // (no overflow)
    }
    if (n_in > FRZ_WHERE_MAX_IN) return frz_fail(FRZ_ERR_UNSUPPORTED, "more than %d set values", FRZ_WHERE_MAX_IN);
    for (uint64_t j = 0; j < n_clauses; j++)
        for (uint64_t v = 0; v < clauses[j].n_in; v++)
            if (clauses[j].in[v] == FRZ_ATTR_NULL)
                return frz_fail(FRZ_ERR_INVALID_ARG, "set value %llu of clause %llu is FRZ_ATTR_NULL", (unsigned long long)v, (unsigned long long)j);
    for (uint64_t j = 0; j < n_clauses; j++)
        if (clauses[j].attr->corpus != s->corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "the attribute was made on another corpus");
    if (base && base->corpus != s->corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "the base subset was made on another corpus");
    FrzWhereDev w = {};
    std::vector<int64_t> sets;
    for (uint64_t j = 0; j < n_clauses; j++) {
        const frz_where_clause& cl = clauses[j];
        FrzWhereClauseDev& d = w.clauses[j];
        d.values = cl.attr->values.get();
        d.n_values = cl.attr->values.cap();
        d.lo = cl.lo;
        d.hi = cl.hi;
        d.in_off = (uint32_t)sets.size();
        d.n_in = cl.n_in ? frz_where_pack_set(cl.in, cl.n_in, sets) : 0;
        d.negate = cl.negate != 0;
    }
    w.n_clauses = (uint32_t)n_clauses;
    FRZ_TRY(frz_ensure_device(s->corpus->st.device));
    return where_fill(s, w, sets, base);
}

// ---------------------------------------------------------------------------------- single-query list calls
namespace {
constexpr uint64_t kNoQuery = UINT64_MAX;   // the check is of a single call: its message names no query

// The handles of one query: the optional subset, boost, groups with their per-group cap, and attribute with its order.
struct CallHandles {
    const frz_subset* s = nullptr;
    const frz_boost* b = nullptr;
    const frz_groups* g = nullptr;
    uint64_t per_group = 1;
    const frz_attr* a = nullptr;
    uint32_t order = 0;
};

// per_group is 1..kFrzCollapseMaxPerGroup, or UINT64_MAX for no cap
frz_status check_per_group(uint64_t per_group, uint64_t query = kNoQuery) {
    char at[32] = "";
    if (query != kNoQuery) snprintf(at, sizeof at, " at %llu", (unsigned long long)query);
    if (per_group == 0) return frz_fail(FRZ_ERR_INVALID_ARG, "per_group = 0%s", at);
    if (per_group > kFrzCollapseMaxPerGroup && per_group != UINT64_MAX)
        return frz_fail(FRZ_ERR_UNSUPPORTED, "per_group = %llu%s: at most %llu rows per group, or UINT64_MAX for no cap",
                        (unsigned long long)per_group, at, (unsigned long long)kFrzCollapseMaxPerGroup);
    return FRZ_OK;
}

// Every handle of a query was made on one of `mine`: the call's corpus, or for a column call any of its columns
// (membership, boosts, group ids and values are by index, so a handle of any column serves every column).  The first that
// was not is reported, in the order subset, boost, groups, attribute; made_on names `mine` in the message.
constexpr const char* kAnotherCorpus = "another corpus";
constexpr const char* kNoColumn = "none of the columns";
frz_status check_handles(const CallHandles& h, const frz_corpus* const* mine, uint64_t n_mine, const char* made_on,
                         uint64_t query = kNoQuery) {
    const auto foreign = [&](const auto* handle) { return handle && std::find(mine, mine + n_mine, handle->corpus) == mine + n_mine; };
    const char* what = foreign(h.s) ? "subset" : foreign(h.b) ? "boost" : foreign(h.g) ? "groups" : foreign(h.a) ? "attribute" : nullptr;
    if (!what) return FRZ_OK;
    char of[40] = "";
    if (query != kNoQuery) snprintf(of, sizeof of, " of query %llu", (unsigned long long)query);
    return frz_fail(FRZ_ERR_INVALID_ARG, "the %s%s %s made on %s", what, of, strcmp(what, "groups") == 0 ? "were" : "was", made_on);
}

// The list call of a query whose arguments have passed, on the corpus's device: the matcher's sort strategy, the first k
// rows, the subset's rows built against `corpus` (subset_scope), the boost as a ranking (with an attribute, as part of the
// order key instead: order_plan.cuh) and the groups as a collapse.
frz_status resolve_call(frz_matcher* m, const frz_corpus* corpus, const CallHandles& h, uint64_t k, ListCall* call) {
    FRZ_TRY(frz_ensure_device(corpus->st.device));
    call->sort = m->config.sort;
    call->limit = k;
    if (h.s) FRZ_TRY(subset_scope(m, corpus, *h.s, nullptr, &call->scope));
    if (h.a) {
        FrzOrderDev o{};
        o.values = h.a->values.get();
        o.n_values = h.a->values.cap();
        o.boost = h.b ? h.b->values.get() : nullptr;
        o.n_boost = h.b ? (uint32_t)h.b->values.cap() : 0;
        o.order = h.order;
        call->ord = Ordering{o};
    } else if (h.b) {
        call->rank = Ranking{h.b->values.get(), (uint32_t)h.b->values.cap(), (uint32_t)h.b->max_set};
    }
    if (h.g) call->col = Collapse{h.g->values.get(), h.g->values.cap(), h.g->n_groups, h.per_group};
    return FRZ_OK;
}

// A single-query call whose arguments have passed (and every query of a batched call that runs on its own): its list
// call, run, the first min(k, total) rows → out.
frz_status list_call(frz_matcher* m, const frz_corpus* corpus, const CallHandles& h, uint64_t k, frz_match* out, uint64_t cap,
                     uint64_t* n_out, uint64_t* n_total, uint32_t* group_counts = nullptr) {
    ListCall call;
    FRZ_TRY(resolve_call(m, corpus, h, k, &call));
    call.group_counts = group_counts;
    return match_list_host(m, corpus, call, out, cap, n_out, n_total);
}
}  // namespace

extern "C" frz_status frz_match_list(frz_matcher* m, const frz_corpus* corpus, frz_match* out, uint64_t cap, uint64_t* n_out) {
    if (!m || !corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    return list_call(m, corpus, CallHandles(), UINT64_MAX, out, cap, n_out, nullptr);
}

extern "C" frz_status frz_match_list_top(frz_matcher* m, const frz_corpus* corpus, uint64_t k, frz_match* out, uint64_t* n_out,
                                         uint64_t* n_total) {
    if (!m || !corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    return list_call(m, corpus, CallHandles(), k, out, k, n_out, n_total);
}

extern "C" frz_status frz_match_list_subset(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, frz_match* out, uint64_t cap,
                                            uint64_t* n_out) {
    if (!m || !corpus || !s) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    const CallHandles h{s};
    FRZ_TRY(check_handles(h, &corpus, 1, kAnotherCorpus));
    return list_call(m, corpus, h, UINT64_MAX, out, cap, n_out, nullptr);
}

extern "C" frz_status frz_match_list_subset_top(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, uint64_t k, frz_match* out,
                                                uint64_t* n_out, uint64_t* n_total) {
    if (!m || !corpus || !s) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    const CallHandles h{s};
    FRZ_TRY(check_handles(h, &corpus, 1, kAnotherCorpus));
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    return list_call(m, corpus, h, k, out, k, n_out, n_total);
}

extern "C" frz_status frz_match_list_ranked(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, const frz_boost* b,
                                            uint64_t k, frz_match* out, uint64_t* n_out, uint64_t* n_total) {
    if (!m || !corpus || !b) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    const CallHandles h{s, b};
    FRZ_TRY(check_handles(h, &corpus, 1, kAnotherCorpus));
    return list_call(m, corpus, h, k, out, k, n_out, n_total);
}

static_assert(FRZ_ORDER_SCORE_THEN_ATTR_DESC == kFrzOrderScoreFirst && FRZ_ORDER_SCORE_THEN_ATTR_ASC + 1 == kFrzOrderCount &&
                  (FRZ_ORDER_ATTR_ASC & 1) && (FRZ_ORDER_SCORE_THEN_ATTR_ASC & 1) && !(FRZ_ORDER_ATTR_DESC & 1),
              "order_plan.cuh mirrors frz_cuda.h");

namespace {
frz_status check_order(uint32_t order, uint64_t query = kNoQuery) {
    char at[32] = "";
    if (query != kNoQuery) snprintf(at, sizeof at, " at %llu", (unsigned long long)query);
    if (order >= kFrzOrderCount) return frz_fail(FRZ_ERR_INVALID_ARG, "order %u%s (at most %u)", order, at, kFrzOrderCount - 1);
    return FRZ_OK;
}
}  // namespace

extern "C" frz_status frz_match_list_ordered(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, const frz_boost* b,
                                             const frz_attr* a, uint32_t order, uint64_t k, frz_match* out, uint64_t* n_out,
                                             uint64_t* n_total) {
    if (!m || !corpus || !a) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    FRZ_TRY(check_order(order));
    const CallHandles h{s, b, nullptr, 1, a, order};
    FRZ_TRY(check_handles(h, &corpus, 1, kAnotherCorpus));
    return list_call(m, corpus, h, k, out, k, n_out, n_total);
}

// The ordered list collapsed by group (DESIGN.md §4.15.1): resolve_call gives the ListCall both an Ordering and a Collapse,
// and collapse_list then ranks the rounds by the order key.
extern "C" frz_status frz_match_list_ordered_collapsed(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, const frz_boost* b,
                                                       const frz_attr* a, uint32_t order, const frz_groups* g, uint64_t per_group,
                                                       uint64_t k, frz_match* out, uint64_t* n_out, uint64_t* n_total,
                                                       uint32_t* group_counts) {
    if (!m || !corpus || !a || !g) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(check_per_group(per_group));
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    FRZ_TRY(check_order(order));
    const CallHandles h{s, b, g, per_group, a, order};
    FRZ_TRY(check_handles(h, &corpus, 1, kAnotherCorpus));
    return list_call(m, corpus, h, k, out, k, n_out, n_total, group_counts);
}

extern "C" frz_status frz_match_list_collapsed(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, const frz_boost* b,
                                               const frz_groups* g, uint64_t per_group, uint64_t k, frz_match* out, uint64_t* n_out,
                                               uint64_t* n_total, uint32_t* group_counts) {
    if (!m || !corpus || !g) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(check_per_group(per_group));
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    const CallHandles h{s, b, g, per_group};
    FRZ_TRY(check_handles(h, &corpus, 1, kAnotherCorpus));
    return list_call(m, corpus, h, k, out, k, n_out, n_total, group_counts);
}

// ---------------------------------------------------------------------------------- column calls
namespace {
// The column set of a column call: at least one column, no null matcher or corpus, every column on one device and of one
// length (one index space) within the u32 index range, and `sort` a strategy.  The matchers are ms[c] (frz_match_list_columns,
// batch_q == nullptr), or *batch_q queries' ms[j * n_cols + c] (frz_match_list_batch_columns).
frz_status check_columns(frz_matcher* const* ms, const frz_corpus* const* cols, uint64_t n_cols, uint8_t sort, const uint64_t* batch_q) {
    if (n_cols == 0) return frz_fail(FRZ_ERR_INVALID_ARG, "n_cols = 0: a columns call needs at least one column");
    if (!ms || !cols) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (!batch_q) {
        for (uint64_t c = 0; c < n_cols; c++)
            if (!ms[c] || !cols[c]) return frz_fail(FRZ_ERR_INVALID_ARG, "null matcher or corpus of column %llu", (unsigned long long)c);
    } else {
        const uint64_t q = *batch_q;
        for (uint64_t c = 0; c < n_cols; c++)
            if (!cols[c]) return frz_fail(FRZ_ERR_INVALID_ARG, "null corpus of column %llu", (unsigned long long)c);
        if (q > UINT64_MAX / n_cols || q * n_cols > SIZE_MAX / sizeof(frz_matcher*))
            return frz_fail(FRZ_ERR_INVALID_ARG, "q * n_cols overflows: q = %llu, n_cols = %llu", (unsigned long long)q, (unsigned long long)n_cols);
        for (uint64_t i = 0; i < q * n_cols; i++)
            if (!ms[i])
                return frz_fail(FRZ_ERR_INVALID_ARG, "null matcher of query %llu, column %llu", (unsigned long long)(i / n_cols),
                                (unsigned long long)(i % n_cols));
    }
    const FrzCorpusStorage& first = cols[0]->st;
    for (uint64_t c = 1; c < n_cols; c++) {
        if (cols[c]->st.device != first.device)
            return frz_fail(FRZ_ERR_INVALID_ARG, "column %llu is on device %d, column 0 on device %d", (unsigned long long)c,
                            cols[c]->st.device, first.device);
        if (cols[c]->st.n != first.n)
            return frz_fail(FRZ_ERR_INVALID_ARG, "column %llu holds %llu rows, column 0 holds %llu: the columns must share one index space",
                            (unsigned long long)c, (unsigned long long)cols[c]->st.n, (unsigned long long)first.n);
    }
    FRZ_TRY(frz_check_index_range(first.n, 0));
    if (sort > FRZ_SORT_INDEX_DESC) return frz_fail(FRZ_ERR_INVALID_ARG, "sort = %u is not a sort strategy", (unsigned)sort);
    return FRZ_OK;
}

// A column call whose arguments have passed (frz_match_list_columns, frz_match_list_columns_ordered): its Columns, its list
// call from the handles, run on ms[0]'s workspace, the first min(k, total) rows → out.
frz_status columns_call(frz_matcher* const* ms, const frz_corpus* const* cols, uint64_t n_cols, uint8_t sort, const CallHandles& h,
                        uint64_t k, frz_match* out, uint64_t* n_out, uint64_t* n_total, uint32_t* group_counts) {
    FRZ_TRY(frz_ensure_device(cols[0]->st.device));   // (before a matcher is read)
    // the list starts from the column of the first non-negated pattern (its base, scanned in full), else from column 0
    Columns cs;
    uint64_t start = n_cols;
    for (uint64_t c = 0; c < n_cols; c++) {
        for (const Compiled& p : ms[c]->compiled) {
            cs.pats.push_back(ColumnPattern{&p, ms[c], &cols[c]->st});
            if (!p.negated && start == n_cols) start = c;
        }
        cs.any_compiled |= !ms[c]->compiled.empty();
    }
    if (start == n_cols) start = 0;
    for (uint64_t c = 0; c < n_cols; c++) {   // the other columns' removed rows (none: no extra launch)
        const FrzCorpusStorage* st = &cols[c]->st;
        if (cols[c] != cols[start] && st->n_removed && std::find(cs.live.begin(), cs.live.end(), st) == cs.live.end())
            cs.live.push_back(st);
    }
    ListCall call;
    FRZ_TRY(resolve_call(ms[0], cols[start], h, k, &call));
    call.sort = sort;
    call.cols = std::move(cs);
    call.group_counts = group_counts;
    return match_list_host(ms[0], cols[start], call, out, k, n_out, n_total);
}
}  // namespace

// Several text fields of the same rows, one matcher per field (DESIGN.md §4.13): the multi-pattern loop over every
// column's patterns in column order, each against its own column (match_patterns), then the ranked, collapsed and top-K
// steps of the single-corpus calls.
extern "C" frz_status frz_match_list_columns(frz_matcher* const* ms, const frz_corpus* const* cols, uint64_t n_cols, uint8_t sort,
                                             const frz_subset* s, const frz_boost* b, const frz_groups* g, uint64_t per_group,
                                             uint64_t k, frz_match* out, uint64_t* n_out, uint64_t* n_total, uint32_t* group_counts) {
    FRZ_TRY(check_columns(ms, cols, n_cols, sort, nullptr));
    if (g) FRZ_TRY(check_per_group(per_group));
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    const CallHandles h{s, b, g, per_group};
    FRZ_TRY(check_handles(h, cols, n_cols, kNoColumn));
    return columns_call(ms, cols, n_cols, sort, h, k, out, n_out, n_total, group_counts);
}

// frz_match_list_columns' joined list ordered by an attribute, then collapsed when groups are given (DESIGN.md §4.15.1).
extern "C" frz_status frz_match_list_columns_ordered(frz_matcher* const* ms, const frz_corpus* const* cols, uint64_t n_cols, uint8_t sort,
                                                     const frz_subset* s, const frz_boost* b, const frz_attr* a, uint32_t order,
                                                     const frz_groups* g, uint64_t per_group, uint64_t k, frz_match* out,
                                                     uint64_t* n_out, uint64_t* n_total, uint32_t* group_counts) {
    FRZ_TRY(check_columns(ms, cols, n_cols, sort, nullptr));
    if (!a) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    if (g) FRZ_TRY(check_per_group(per_group));
    if (!out && k > 0) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    FRZ_TRY(check_order(order));
    const CallHandles h{s, b, g, per_group, a, order};
    FRZ_TRY(check_handles(h, cols, n_cols, kNoColumn));
    return columns_call(ms, cols, n_cols, sort, h, k, out, n_out, n_total, group_counts);
}

// ---------------------------------------------------------------------------------- batched top-K: entry points
extern "C" frz_status frz_match_list_batch(frz_matcher* const* ms, uint64_t q, const frz_corpus* corpus,
                                           const frz_subset* const* subsets, const frz_boost* const* boosts, uint64_t k,
                                           frz_match* out, uint64_t* n_out, uint64_t* n_total) {
    return frz_match_list_batch_collapsed(ms, q, corpus, subsets, boosts, nullptr, nullptr, k, out, n_out, n_total, nullptr);
}

extern "C" frz_status frz_match_list_batch_collapsed(frz_matcher* const* ms, uint64_t q, const frz_corpus* corpus,
                                                     const frz_subset* const* subsets, const frz_boost* const* boosts,
                                                     const frz_groups* const* groups, const uint64_t* per_group, uint64_t k,
                                                     frz_match* out, uint64_t* n_out, uint64_t* n_total, uint32_t* const* group_counts) {
    return frz_match_list_batch_ordered(ms, q, corpus, subsets, boosts, nullptr, nullptr, groups, per_group, k, out, n_out, n_total,
                                        group_counts);
}

namespace {
// The arguments of a batched call (frz_match_list_batch_ordered, frz_match_list_batch_columns).  bc: a column call,
// whose query j has the matchers ms[j * n_cols ..] and whose corpus is its column 0 (it has no attributes).
struct BatchCall {
    frz_matcher* const* ms;
    uint64_t q;
    const frz_corpus* corpus;
    const BatchColumns* bc;
    const frz_subset* const* subsets;
    const frz_boost* const* boosts;
    const frz_groups* const* groups;
    const uint64_t* per_group;
    uint64_t k;
    frz_match* out;
    uint64_t* n_out;
    uint64_t* n_total;
    uint32_t* const* group_counts;
    const frz_attr* const* attrs = nullptr;
    const uint32_t* orders = nullptr;   // nullptr: FRZ_ORDER_ATTR_DESC for every query

    CallHandles handles_of(uint64_t j) const {
        return CallHandles{subsets ? subsets[j] : nullptr, boosts ? boosts[j] : nullptr, groups ? groups[j] : nullptr,
                           per_group ? per_group[j] : 1, attrs ? attrs[j] : nullptr, orders ? orders[j] : (uint32_t)FRZ_ORDER_ATTR_DESC};
    }
};

// The driver of the batched calls once their matchers and columns have passed: every query's per_group (with or without
// groups), every order (with or without an attribute) and the handles, then the outputs, are checked; the queries of the
// batched class run in sub-batches (batch_run), the ordered ones in sub-batches of their own, every other query, and every
// query of an overflowed sub-batch, its single-query call.
frz_status batch_drive(const BatchCall& a) {
    frz_matcher* const* ms = a.ms;
    const uint64_t q = a.q, k = a.k;
    const frz_corpus* corpus = a.corpus;
    const BatchColumns* bc = a.bc;
    frz_match* out = a.out;
    uint64_t* n_out = a.n_out;
    uint64_t* n_total = a.n_total;
    for (uint64_t j = 0; a.per_group && j < q; j++) FRZ_TRY(check_per_group(a.per_group[j], j));
    for (uint64_t j = 0; a.orders && j < q; j++) FRZ_TRY(check_order(a.orders[j], j));
    for (uint64_t j = 0; j < q; j++)
        FRZ_TRY(bc ? check_handles(a.handles_of(j), bc->cols, bc->n_cols, kNoColumn, j) : check_handles(a.handles_of(j), &corpus, 1, kAnotherCorpus, j));
    if (q && !n_out) return frz_fail(FRZ_ERR_INVALID_ARG, "null n_out");
    if (k && (q > UINT64_MAX / k || q * k > SIZE_MAX / sizeof(frz_match)))
        return frz_fail(FRZ_ERR_INVALID_ARG, "q * k overflows: q = %llu, k = %llu", (unsigned long long)q, (unsigned long long)k);
    if (q * k > 0 && !out) return frz_fail(FRZ_ERR_INVALID_ARG, "null out");
    if (q == 0) return FRZ_OK;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
        cudaGetLastError();
        return frz_fail(FRZ_ERR_NO_DEVICE, "no CUDA device available; this library has no CPU fallback");
    }
    FRZ_TRY(frz_ensure_device(corpus->st.device));
    const FrzCorpusStorage& cs = corpus->st;
    FRZ_TRY(frz_check_index_range(cs.n, 0));
    for (uint64_t& v : g_batch_last) v = 0;
    auto counts_of = [&](uint64_t j) { return a.group_counts ? a.group_counts[j] : nullptr; };
    auto single = [&](uint64_t j) {
        frz_match* oj = k ? out + j * k : nullptr;
        uint64_t* tj = n_total ? &n_total[j] : nullptr;
        const CallHandles h = a.handles_of(j);
        if (bc)
            return frz_match_list_columns(ms + j * bc->n_cols, bc->cols, bc->n_cols, bc->sort, h.s, h.b, h.g, h.per_group, k, oj,
                                          &n_out[j], tj, counts_of(j));
        return list_call(ms[j], corpus, h, k, oj, k, &n_out[j], tj, counts_of(j));
    };
    auto selected = [&](uint64_t j) {
        return bc ? batch_columns_selected(ms + j * bc->n_cols, *bc) : batchable(ms[j], cs) && batch_selected(ms[j], cs);
    };
    std::vector<uint64_t> batched;
    const uint64_t cap = batch_survivor_cap(cs);
    const uint64_t list_rows = std::max<uint64_t>(cs.n, 1);
    const uint64_t base = BatchLayout::per_query(cs, k, cap) + (bc ? frz_batch_columns_bytes(bc->n_cols, list_rows, sizeof(FrzPatternDev)) : 0);
    const uint64_t fit = k <= kFrzBatchMaxK ? kBatchScratchBytes / base : 0;
    const uint64_t qs_max = std::min<uint64_t>(fit, kFrzBatchMaxSub);
    uint64_t n_groups_max = 0;   // the largest n_groups among the batched grouped queries
    for (uint64_t j = 0; j < q; j++) {
        const CallHandles h = a.handles_of(j);
        const uint64_t n_groups = h.g ? h.g->n_groups : 0;
        if (qs_max >= 2 && selected(j) &&
            (!h.g || (frz_batch_collapse_fit(kBatchScratchBytes, base, n_groups, list_rows) &&
                      (!counts_of(j) || n_groups <= kBatchMaxCountedGroups))) &&
            (!h.a || frz_batch_order_fit(kBatchScratchBytes, base, n_groups, list_rows))) {
            batched.push_back(j);
            n_groups_max = std::max(n_groups_max, n_groups);
        } else {
            FRZ_TRY(single(j));
        }
    }
    if (batched.size() < std::max<uint64_t>(2, g_batch_min_queries.load())) {   // a few queries cost what a loop of single calls costs
        for (uint64_t j : batched) FRZ_TRY(single(j));
        return FRZ_OK;
    }
    // the ordered queries go to sub-batches of their own; when their tables do not fit two to a sub-batch beside the
    // call's largest group tables, they run their single-query calls
    std::vector<uint64_t> ordered, unordered;
    for (uint64_t j : batched) (a.handles_of(j).a ? ordered : unordered).push_back(j);
    if (!ordered.empty() && !frz_batch_order_fit(kBatchScratchBytes, base, n_groups_max, list_rows)) {
        for (uint64_t j : ordered) FRZ_TRY(single(j));
        ordered.clear();
    }
    // every query's subset and boost, as k_batch_top<ScopedKey> reads them (none when no query has either); an ordered
    // query's subset is read by k_batch_order_members, its boost is part of its order key
    std::vector<FrzBatchScope> scopes;
    for (uint64_t j : batched) {
        const CallHandles h = a.handles_of(j);
        if (!h.s && !h.b) continue;
        if (scopes.empty()) scopes.resize(q);
        FrzBatchScope& r = scopes[j];
        if (h.s) {
            r.scoped = 1;
            r.bits = h.s->bits.get();
            r.n_bits = h.s->n_bits;
        }
        if (h.b) {
            r.ranked = 1;
            r.boost = h.b->values.get();
            r.n_boost = (uint32_t)h.b->values.cap();
        }
    }
    // every query's groups, as the batched collapse reads them (none when no batched query has groups)
    std::vector<FrzBatchCollapse> cols;
    std::vector<uint64_t> n_groups;
    for (uint64_t j : batched) {
        const CallHandles h = a.handles_of(j);
        if (!h.g) continue;
        if (cols.empty()) { cols.resize(q, FrzBatchCollapse()); n_groups.resize(q, 0); }
        FrzBatchCollapse& r = cols[j];
        r.ids = h.g->values.get();
        r.n_ids = h.g->values.cap();
        r.per_group = h.per_group == UINT64_MAX ? 0xFFFFFFFFu : (uint32_t)h.per_group;
        r.order = collapse_order(h.b != nullptr, sort_by_score(bc ? bc->sort : ms[j]->config.sort));
        n_groups[j] = h.g->n_groups;
    }
    BatchGroups gr;
    if (!cols.empty()) {
        gr.cols = cols.data();
        gr.n_groups = n_groups.data();
        gr.counts = a.group_counts;
    }
    // every ordered query's attribute, boost and order (its direction is set per sub-batch)
    std::vector<FrzOrderDev> ords;
    for (uint64_t j : ordered) {
        const CallHandles h = a.handles_of(j);
        if (ords.empty()) ords.resize(q, FrzOrderDev());
        FrzOrderDev& o = ords[j];
        o.values = h.a->values.get();
        o.n_values = h.a->values.cap();
        o.boost = h.b ? h.b->values.get() : nullptr;
        o.n_boost = h.b ? (uint32_t)h.b->values.cap() : 0;
        o.order = h.order;
    }
    uint64_t qs_fit = n_groups_max ? std::min<uint64_t>(frz_batch_collapse_fit(kBatchScratchBytes, base, n_groups_max, list_rows),
                                                        kFrzBatchMaxSub)
                                   : qs_max;
    if (!ordered.empty()) qs_fit = std::min<uint64_t>(qs_fit, frz_batch_order_fit(kBatchScratchBytes, base, n_groups_max, list_rows));
    const uint64_t qs = std::min<uint64_t>(qs_fit, std::max(ordered.size(), unordered.size()));
    const BatchLayout L(cs, k, cap, qs, n_groups_max, bc ? bc->n_cols : 0, !ordered.empty());
    FrzDevArray<uint8_t> scratch;   // released when the call returns
    FRZ_TRY(scratch.reserve(L.bytes));
    if (L.groups)   // the round tables start zero, and every sub-batch's rounds leave them zero
        FRZ_CUDA_TRY(cudaMemsetAsync(scratch.get() + L.off[BatchLayout::BEST], 0, L.off[BatchLayout::TAKEN] - L.off[BatchLayout::BEST]));
    if (L.groups && L.ordered)   // the ordered rounds' second table too
        FRZ_CUDA_TRY(cudaMemsetAsync(scratch.get() + L.off[BatchLayout::BESTLO], 0, L.off[BatchLayout::END] - L.off[BatchLayout::BESTLO]));
    for (const std::vector<uint64_t>* part : {&unordered, &ordered}) {
        const FrzOrderDev* po = part == &ordered ? ords.data() : nullptr;
        for (uint64_t s = 0; s < part->size(); s += qs) {
            const uint32_t ns = (uint32_t)std::min<uint64_t>(qs, part->size() - s);
            bool overflow = false;
            FrzLaunchStats st;
            FRZ_TRY(batch_run(ms, scopes.empty() ? nullptr : scopes.data(), gr, part->data() + s, ns, corpus, k, L, scratch.get(), out,
                              n_out, n_total, &overflow, st, bc, po));
            g_batch_last[overflow ? 1 : 0] += ns;
            g_batch_last[2]++;
            g_batch_last[3] += st.launches;
            if (overflow)   // the single-query pipeline retries with worst-case lists
                for (uint32_t j = 0; j < ns; j++) FRZ_TRY(single((*part)[s + j]));
        }
    }
    return FRZ_OK;
}

}  // namespace

// Query j is frz_match_list_ordered_collapsed(ms[j], corpus, subsets[j], boosts[j], attrs[j], orders[j], groups[j],
// per_group[j], ...) with an attribute and groups, frz_match_list_ordered(...) with an attribute alone, and query j of
// frz_match_list_batch_collapsed without one.  Its batched class orders its rows on the device (batch_run, order.cu).
extern "C" frz_status frz_match_list_batch_ordered(frz_matcher* const* ms, uint64_t q, const frz_corpus* corpus,
                                                   const frz_subset* const* subsets, const frz_boost* const* boosts,
                                                   const frz_attr* const* attrs, const uint32_t* orders, const frz_groups* const* groups,
                                                   const uint64_t* per_group, uint64_t k, frz_match* out, uint64_t* n_out,
                                                   uint64_t* n_total, uint32_t* const* group_counts) {
    if (!ms || !corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    for (uint64_t j = 0; j < q; j++)
        if (!ms[j]) return frz_fail(FRZ_ERR_INVALID_ARG, "null matcher at %llu", (unsigned long long)j);
    return batch_drive(BatchCall{ms, q, corpus, nullptr, subsets, boosts, groups, per_group, k, out, n_out, n_total, group_counts, attrs,
                                 orders});
}

// Query j is frz_match_list_columns(ms + j * n_cols, cols, n_cols, sort, subsets[j], boosts[j], groups[j], per_group[j], ...);
// its batched class joins its columns on the device (batch_run, batch_columns.cu).
extern "C" frz_status frz_match_list_batch_columns(frz_matcher* const* ms, uint64_t q, const frz_corpus* const* cols, uint64_t n_cols,
                                                   uint8_t sort, const frz_subset* const* subsets, const frz_boost* const* boosts,
                                                   const frz_groups* const* groups, const uint64_t* per_group, uint64_t k,
                                                   frz_match* out, uint64_t* n_out, uint64_t* n_total, uint32_t* const* group_counts) {
    FRZ_TRY(check_columns(ms, cols, n_cols, sort, &q));
    const BatchColumns bc{cols, n_cols, sort};
    return batch_drive(BatchCall{ms, q, cols[0], &bc, subsets, boosts, groups, per_group, k, out, n_out, n_total, group_counts});
}

extern "C" frz_status frz_match_list_batch_top(frz_matcher* const* ms, uint64_t q, const frz_corpus* corpus, uint64_t k, frz_match* out,
                                               uint64_t* n_out, uint64_t* n_total) {
    return frz_match_list_batch(ms, q, corpus, nullptr, nullptr, k, out, n_out, n_total);
}

extern "C" frz_status frz_match_list_into(frz_matcher* m, const frz_corpus* corpus, uint32_t index_offset, frz_match* out,
                                          uint64_t cap, uint64_t* n_out) {
    if (!m || !corpus) return frz_fail(FRZ_ERR_INVALID_ARG, "null argument");
    FRZ_TRY(frz_ensure_device(corpus->st.device));
    ListCall call;
    call.index_offset = index_offset;
    return match_list_host(m, corpus, call, out, cap, n_out, nullptr);
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
        ListCall call;
        call.sort = m->config.sort;
        call.limit = limit;
        call.index_offset = index_offset;
        call.final_out = reinterpret_cast<FrzMatchDev*>(d_out);
        FrzMatchDev* d_list = nullptr;
        return match_list_device(m, shard->st, call, &d_list, stream, st);
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
        FRZ_TRY(needle_table(m, pat, m->ws.device, &x.ntab));   // a synchronous upload, so before the first H2D chunk
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
