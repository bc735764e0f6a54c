/*
 * frz_cuda.h — C ABI of the H100-native `match_list` path of saghen/frizbee.
 *
 * This header is the drop-in boundary (SURVEY.md §8(b)).  Every entry point
 * names the reference interface it replaces (paths relative to the reference
 * crate root).  Plain pointers and sizes only: no torch, no C++ types.
 *
 * Reference interfaces replaced:
 *   trait Specialized::match_list            src/matcher/algo.rs:14-22
 *   Matcher::{new,from_patterns,from_query}  src/matcher/mod.rs:90-136
 *   Matcher::match_list                      src/matcher/mod.rs:212-222
 *     (and, truncated to its first k rows, frz_match_list_top / frz_match_list_parallel*_top)
 *   Matcher::match_list_parallel             src/matcher/parallel.rs:18-89
 *   Pattern::{parse,parse_query}             src/pattern.rs:100-222
 *   radix_sort_matches                       src/sort.rs:6-40
 *   Match / Config / Scoring / enums         src/lib.rs:141-153,236-271,313-323,439-478
 *
 * There is NO CPU fallback behind this ABI: every compute entry point fails
 * with FRZ_ERR_NO_DEVICE / FRZ_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef FRZ_CUDA_H
#define FRZ_CUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FRZ_ABI_VERSION 3
#if defined(__GNUC__)
#define FRZ_API __attribute__((visibility("default")))
#else
#define FRZ_API
#endif

/* ------------------------------------------------------------------ status */

typedef enum frz_status {
    FRZ_OK = 0,
    FRZ_ERR_INVALID_ARG = 1,
    /* reference panics: "needle too long and could overflow the u16 score" (src/lib.rs:524-527) */
    FRZ_ERR_NEEDLE_TOO_LONG = 2,
    /* reference panics: "gap penalties too large" (src/lib.rs:532-536) */
    FRZ_ERR_GAP_OVERFLOW = 3,
    /* reference panics: "too many items in haystack, will overflow the u32 index" (src/matcher/mod.rs:438-446) */
    FRZ_ERR_TOO_MANY_ITEMS = 4,
    /* reference panics: "threads must be positive" (src/matcher/parallel.rs:24) */
    FRZ_ERR_THREADS_ZERO = 5,
    /* caller-provided output buffer too small; *n_out holds the required count */
    FRZ_ERR_CAPACITY = 6,
    FRZ_ERR_CUDA = 7,
    FRZ_ERR_NO_DEVICE = 8,
    /* feature of the reference not built on the GPU path yet (never a silent CPU fallback): needles over 1024 bytes,
     * needles over 64 bytes on the unicode path or in frz_match_indices, max_typos > 15 below
     * the needle length (DESIGN.md §7) */
    FRZ_ERR_UNSUPPORTED = 9,
    FRZ_ERR_OOM = 10,
    /* NCCL missing / failed, or a peer rank did not answer (multi-GPU entry points only) */
    FRZ_ERR_NCCL = 11
} frz_status;

/* thread-local, human-readable detail for the last non-OK status */
FRZ_API const char* frz_last_error(void);
FRZ_API const char* frz_status_str(frz_status s);
FRZ_API int frz_abi_version(void);

/* ------------------------------------------------------------------- types */

/* `Match` (src/lib.rs:141-153).  The reference struct is default-repr Rust; the shim converts. */
typedef struct frz_match {
    uint32_t index; /* index in the original haystack list (+ index_offset) */
    uint16_t score;
    uint8_t exact;  /* 0/1 */
    uint8_t _pad;   /* always 0 */
} frz_match;

/* `Scoring` (src/lib.rs:439-478), defaults from src/const.rs:1-10 */
typedef struct frz_scoring {
    uint16_t match_score;          /* 12 */
    uint16_t mismatch_penalty;     /*  6 */
    uint16_t gap_open_penalty;     /*  5 */
    uint16_t gap_extend_penalty;   /*  1 */
    uint16_t prefix_bonus;         /* 12 */
    uint16_t capitalization_bonus; /*  4 */
    uint16_t matching_case_bonus;  /*  4 */
    uint16_t exact_match_bonus;    /*  8 */
    uint16_t delimiter_bonus;      /*  4 */
} frz_scoring;

/* `CaseMatching` (src/lib.rs:353-377) */
enum { FRZ_CASE_IGNORE = 0, FRZ_CASE_SMART = 1, FRZ_CASE_RESPECT = 2 };
/* `UnicodeMatching` (src/lib.rs:379-402) */
enum { FRZ_UNICODE_IGNORE = 0, FRZ_UNICODE_SMART = 1, FRZ_UNICODE_ALWAYS = 2 };
/* `Matching` (src/lib.rs:413-436) */
enum { FRZ_MATCHING_FUZZY = 0, FRZ_MATCHING_EXACT = 1, FRZ_MATCHING_PREFIX = 2,
       FRZ_MATCHING_SUFFIX = 3, FRZ_MATCHING_SUBSTRING = 4 };
/* `SortStrategy` (src/lib.rs:311-351) */
enum { FRZ_SORT_SCORE_THEN_INDEX_ASC = 0, FRZ_SORT_SCORE_THEN_INDEX_DESC = 1,
       FRZ_SORT_INDEX_ASC = 2, FRZ_SORT_INDEX_DESC = 3 };

#define FRZ_MAX_TYPOS_NONE (-1)

/* `Config` (src/lib.rs:236-271) */
typedef struct frz_config {
    int32_t max_typos;     /* FRZ_MAX_TYPOS_NONE (= Rust `None`) or 0..65535; default 0 */
    uint8_t casing;        /* FRZ_CASE_*;     default SMART */
    uint8_t unicode;       /* FRZ_UNICODE_*;  default SMART */
    uint8_t matching;      /* FRZ_MATCHING_*; default FUZZY */
    uint8_t sort;          /* FRZ_SORT_*;     default SCORE_THEN_INDEX_ASC */
    frz_scoring scoring;
    /* Which reference SIMD backend the integer results are bit-exact with
     * (SURVEY.md §8 finding 1: scores depend on the lane count).
     * 0 = auto: the backend `Matcher::get_backend` (src/matcher/mod.rs:448-498)
     * would select on THIS host's CPU; else 16 (SSE/NEON/scalar), 32 (AVX2),
     * 64 (AVX-512+VBMI) = lane count of the u8 family; the u16 family
     * (needle too long for u8 scores) uses half of it. */
    uint8_t emulate_lanes;
    uint8_t _pad;
} frz_config;

/* `Pattern` + `PatternConfig` (src/pattern.rs:9-18, 230-246).  Overrides use -1 = inherit. */
typedef struct frz_pattern {
    const uint8_t* needle;
    size_t needle_len;
    uint8_t negated;
    uint8_t has_scoring;       /* 1 → `scoring` overrides Config::scoring */
    int8_t casing;             /* -1 inherit, else FRZ_CASE_* */
    int8_t unicode;            /* -1 inherit, else FRZ_UNICODE_* */
    int8_t matching;           /* -1 inherit, else FRZ_MATCHING_* */
    int8_t _pad[3];
    int32_t max_typos;         /* -1 inherit (PatternConfig cannot express "unlimited"), else 0..65535 */
    frz_scoring scoring;
} frz_pattern;

FRZ_API void frz_config_default(frz_config* out);   /* Config::default()  src/lib.rs:260-271 */
FRZ_API void frz_scoring_default(frz_scoring* out); /* Scoring::default() src/lib.rs:461-478 */

/* ------------------------------------------------------- query-atom parser */

/* Owned parse result of Pattern::parse_query (src/pattern.rs:190-222). */
typedef struct frz_query frz_query;
FRZ_API frz_status frz_parse_query(const uint8_t* query, size_t len, frz_query** out);
/* Pattern::parse (src/pattern.rs:100-165) on one atom; result holds exactly one pattern
 * (even when its needle is empty, as in the reference). */
FRZ_API frz_status frz_parse_atom(const uint8_t* atom, size_t len, frz_query** out);
FRZ_API size_t frz_query_len(const frz_query* q);
/* The returned pattern's `needle` points into `q`; valid until frz_query_destroy. */
FRZ_API frz_status frz_query_get(const frz_query* q, size_t i, frz_pattern* out);
FRZ_API void frz_query_destroy(frz_query* q);

/* ----------------------------------------------------------------- corpus */

/* A haystack list, packed and resident in HBM on one device.  Read-only for matchers (only frz_corpus_append, _remove and
 * _replace mutate it),
 * reusable across matchers/needles (the interactive use: haystacks fixed, needle changes).
 * Replaces the `&[S: AsRef<str>]` argument of Matcher::match_list (src/matcher/mod.rs:212).
 * Input is Arrow-style: `bytes` = concatenated UTF-8, `offsets[n+1]` monotone byte offsets. */
typedef struct frz_corpus frz_corpus;

FRZ_API frz_status frz_corpus_create(const uint8_t* bytes, const uint64_t* offsets, uint64_t n,
                             int device, frz_corpus** out);
/* same, for either Arrow offset width (Utf8 = 4-byte, LargeUtf8 = 8-byte offsets); a sliced array may start at
 * offsets[0] != 0.  The value bytes are streamed host->device in tile-aligned chunks on a copy stream while
 * the bucketing kernels run (SURVEY.md §8(f) rank 1: the step before Matcher::match_list, src/matcher/mod.rs:212). */
FRZ_API frz_status frz_corpus_create_arrow(const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n,
                                   int device, frz_corpus** out);
/* Incremental ingestion: appends n_new haystacks (host Arrow buffers, either offset width); they take the indices
 * [frz_corpus_len, frz_corpus_len + n_new).  Only the partial last tile is re-bucketed.  Synchronous; the caller
 * must not run it concurrently with a match on the same corpus.  (Reference side: the caller pushing onto the
 * Vec<String> it later passes to Matcher::match_list, src/matcher/mod.rs:212.) */
FRZ_API frz_status frz_corpus_append(frz_corpus* c, const uint8_t* bytes, const void* offsets, int offset_width,
                             uint64_t n_new);
/* In-place edits.  (Reference side: the caller removing or rewriting entries of the Vec<String> it later passes to
 * Matcher::match_list, src/matcher/mod.rs:212.)  After any sequence of create / append / remove / replace, every match call
 * on the corpus (frz_match_list, _top, _into, frz_match_indices, frz_match_shard_device, frz_match_list_parallel*) returns
 * what it returns on a fresh corpus of the current list, minus the rows of removed indices, in the same order;
 * frz_match_indices reports a removed row as not matching.  Both calls are synchronous and check every argument on the
 * host before anything changes, so a refused call leaves the corpus as it was; the caller must not run them concurrently
 * with a match on the same corpus.  n == 0 is a no-op that makes no CUDA call.  An index >= frz_corpus_len, or a NULL
 * array with n > 0, is FRZ_ERR_INVALID_ARG.
 *
 * Haystacks which[0..n) stop matching in every call on this corpus.  Indices do not move: frz_corpus_len is unchanged
 * and later appends continue after it.  Removing a removed haystack is a no-op; duplicates in `which` are allowed. */
FRZ_API frz_status frz_corpus_remove(frz_corpus* c, const uint32_t* which, uint64_t n);
/* Haystack which[j] becomes bytes[offsets[j], offsets[j+1]) (Arrow buffers, offset width 4 or 8, host memory); a removed
 * haystack comes back.  Only the tiles holding `which` are re-packed, in one batch, at the end of the packed arena; when
 * the space they leave behind outgrows the live data the arena is compacted into a fresh one (old and new arena are held
 * together while the units move).  The compaction is the last step and only an optimisation: when its arena cannot be
 * allocated the call still succeeds, keeps the dead space and the next edit tries again.  Device memory beyond
 * frz_corpus_device_bytes while the call runs: the touched tiles' raw bytes, the new strings and the touched tiles'
 * metadata (about a second copy of the list when every tile is touched); the corpus keeps this staging for its next edit
 * only while it is under 64 MiB, a larger one is given back when the call returns.
 * A duplicate index is FRZ_ERR_INVALID_ARG, a replacement over 4194302 bytes FRZ_ERR_UNSUPPORTED. */
FRZ_API frz_status frz_corpus_replace(frz_corpus* c, const uint32_t* which, uint64_t n, const uint8_t* bytes,
                                      const void* offsets, int offset_width);
/* same, from a pointer array + lengths (the layout a Rust `&[&str]` has) */
FRZ_API frz_status frz_corpus_create_ptrs(const uint8_t* const* ptrs, const uint32_t* lens, uint64_t n,
                                  int device, frz_corpus** out);
/* same, but `d_bytes`/`d_offsets` are already device pointers on `device`.  As in Arrow, haystack i is
 * d_bytes[d_offsets[i], d_offsets[i+1]): a slice may start at d_offsets[0] != 0, and d_bytes may have any alignment.
 * total_bytes must equal d_offsets[n] - d_offsets[0] (the sum of the lengths, frz_corpus_total_bytes), else
 * FRZ_ERR_INVALID_ARG.  The work runs on `stream` (a cudaStream_t, NULL = the legacy default stream), so that stream must
 * be ordered after whatever wrote the buffers.  Blocking: the corpus is complete when the call returns, and the caller
 * may then reuse or free d_bytes/d_offsets. */
FRZ_API frz_status frz_corpus_create_device(const uint8_t* d_bytes, const uint64_t* d_offsets, uint64_t n,
                                    uint64_t total_bytes, int device, void* stream, frz_corpus** out);
/* Every constructor, frz_corpus_append and the end-to-end calls refuse a haystack longer than 4194302 bytes (4 MiB - 2)
 * with FRZ_ERR_UNSUPPORTED; a refused append leaves the corpus as it was. */
FRZ_API uint64_t frz_corpus_len(const frz_corpus* c);           /* size of the index space (removed indices included) */
FRZ_API uint64_t frz_corpus_total_bytes(const frz_corpus* c);   /* sum of the live (not removed) haystacks' lengths */
FRZ_API uint64_t frz_corpus_device_bytes(const frz_corpus* c);  /* HBM footprint of the packed form (dead arena space included) */
FRZ_API int frz_corpus_device(const frz_corpus* c);
FRZ_API void frz_corpus_destroy(frz_corpus* c);

/* ---------------------------------------------------------------- matcher */

/* `Matcher` (src/matcher/mod.rs:76-188). */
typedef struct frz_matcher frz_matcher;

/* Matcher::from_patterns (src/matcher/mod.rs:105-111); n_patterns == 1 ⇔ Matcher::new */
FRZ_API frz_status frz_matcher_create(const frz_pattern* patterns, size_t n_patterns,
                              const frz_config* config, frz_matcher** out);
/* Matcher::from_query (src/matcher/mod.rs:136-138) */
FRZ_API frz_status frz_matcher_from_query(const uint8_t* query, size_t len, const frz_config* config,
                                  frz_matcher** out);
/* Matcher::set_config (src/matcher/mod.rs:154-160) */
FRZ_API frz_status frz_matcher_set_config(frz_matcher* m, const frz_config* config);
/* `impl Clone for Matcher` (src/matcher/mod.rs:76): same patterns and config, its own device scratch */
FRZ_API frz_status frz_matcher_clone(const frz_matcher* m, frz_matcher** out);
FRZ_API void frz_matcher_destroy(frz_matcher* m);

/* Introspection of what `get_backend` selected for pattern i (src/matcher/mod.rs:448-498):
 * lanes ∈ {8,16,32,64}; score_bits ∈ {8,16}; prefilter_lanes ∈ {16,32,64}; is_literal 0/1. */
FRZ_API frz_status frz_matcher_backend_info(const frz_matcher* m, size_t i, int* lanes, int* score_bits,
                                    int* prefilter_lanes, int* is_literal);
FRZ_API size_t frz_matcher_num_patterns(const frz_matcher* m); /* compiled (non-empty-needle) patterns */

/* Matcher::match_list (src/matcher/mod.rs:212-222): all patterns, ordered per config.sort.
 * `out` is HOST memory with room for `cap` matches.  On FRZ_ERR_CAPACITY *n_out = needed. */
FRZ_API frz_status frz_match_list(frz_matcher* m, const frz_corpus* corpus,
                          frz_match* out, uint64_t cap, uint64_t* n_out);

/* Matcher::match_list (src/matcher/mod.rs:212-222) followed by truncation to its first k rows — the rows a UI shows.
 * The reference has no such method.  Bit-identical to frz_match_list(m, corpus)[0 : min(k, total)] under
 * m->config.sort, for every sort strategy.  `out` is HOST memory with room for `k` matches (room for
 * min(k, frz_corpus_len(corpus)) suffices: no more rows can match); *n_out = min(k, total) and
 * *n_total = total (the full match count; n_total may be NULL).  k = 0 counts and copies nothing.  Never returns
 * FRZ_ERR_CAPACITY; a NULL `out` with k > 0 is FRZ_ERR_INVALID_ARG.  The score sort stores only the first k positions
 * and only min(k, total) matches cross PCIe. */
FRZ_API frz_status frz_match_list_top(frz_matcher* m, const frz_corpus* corpus, uint64_t k,
                              frz_match* out, uint64_t* n_out, uint64_t* n_total);

/* The reference has no such method: Matcher::match_list (src/matcher/mod.rs:212-222) of each of q matchers over one
 * list, each truncated to its first k rows as by frz_match_list_top — many queries against one resident corpus (a fuzzy
 * join, a service answering many users, "did you mean" for a batch of identifiers) in one call.
 * For every j < q, out[j*k .. j*k + n_out[j]), n_out[j] and n_total[j] are bit for bit what frz_match_list_top(ms[j],
 * corpus, k, ...) returns, for every matcher, config and sort strategy; rows out[j*k + n_out[j] .. (j+1)*k) are not
 * written.  `out` is HOST memory with room for q*k matches; n_total may be NULL; k = 0 only counts (out may then be NULL);
 * q = 0 is a no-op that makes no CUDA call.  A NULL ms, any NULL ms[j], a NULL corpus, a NULL n_out with q > 0, a NULL out
 * with q*k > 0, or a q*k that overflows uint64_t or size_t is FRZ_ERR_INVALID_ARG, checked before any device work.  A
 * matcher may appear more than once in ms; the call only reads the matchers' compiled patterns.  Blocking; neither the
 * matchers nor the corpus may be used concurrently by another call.  Never FRZ_ERR_CAPACITY.
 * Queries of one compiled pattern that is fuzzy, not negated, on the byte path and at most 64 bytes long, with k <= 1024,
 * on a corpus of at most 2^18 rows (2^21 for max_typos = 0), when a call has at least 32 of them, run in sub-batches whose every stage covers all
 * of the sub-batch's queries in one launch (per kernel variant present), with one upload, one read-back and one
 * synchronise per sub-batch (DESIGN.md §4.11: where that was measured faster than a loop).  The sub-batch's device scratch has a fixed budget,
 * so the memory a call holds does not grow with q (beyond it: the rows and patterns of a sub-batch); it is released when
 * the call returns.  Every other query (multi-pattern, negated, literal modes, unicode, 65-1024-byte needles, the empty
 * matcher, k > 1024, larger corpora and smaller batches) runs frz_match_list_top's pipeline inside the same call, one
 * after another: correct, but not faster than a loop. */
FRZ_API frz_status frz_match_list_batch_top(frz_matcher* const* ms, uint64_t q, const frz_corpus* corpus, uint64_t k,
                                            frz_match* out, uint64_t* n_out, uint64_t* n_total);
/* Test aid: the corpus-size and query-count limits of the batched path of frz_match_list_batch_top,
 * frz_match_list_batch, frz_match_list_batch_collapsed, frz_match_list_batch_ordered and frz_match_list_batch_columns,
 * process-wide (0 restores
 * a limit's default: 2^18 rows, 32 queries; max_typos = 0 queries batch up to the larger of max_rows and 2^21 rows;
 * fewer than 2 queries never batch).  For frz_match_list_batch_columns, max_rows limits every query, and a query with a
 * typo budget in some column batches only when max_rows is set (by default it runs frz_match_list_columns).  Lets tests reach the batched kernels with
 * small batches and tools/bench_batch.py time the batched path on both sides of the defaults.  Not for concurrent use with
 * batch calls. */
FRZ_API void frz_debug_batch_limits(uint64_t max_rows, uint64_t min_queries);
/* Test aid: what the calling thread's last frz_match_list_batch_top, frz_match_list_batch,
 * frz_match_list_batch_collapsed, frz_match_list_batch_ordered or frz_match_list_batch_columns did: [0] queries answered by
 * the batched kernels, [1] queries of sub-batches whose survivor lists overflowed (answered again by their single-query
 * call's pipeline),
 * [2] sub-batches run, [3] kernel launches of the batched path.  All zero after a call that ran no sub-batch. */
FRZ_API void frz_debug_batch_last(uint64_t out[4]);
/* Test aid: force > 0 makes this thread's frz_subset_where_batch run its batched kernels at every q and corpus length,
 * force == 0 restores its rule (see frz_subset_where_batch), force < 0 changes nothing.  Returns whether this thread's last
 * frz_subset_where_batch ran the batched kernels. */
FRZ_API int frz_debug_where_batch(int force);

/* ---------------------------------------------------------------- subsets
 *
 * A chosen set of rows of a resident corpus, matched without staging them again: a picker scoped to one directory, a
 * history search limited to this session, "search within these results".  (Reference side: the caller passing a
 * smaller slice to Matcher::match_list, src/matcher/mod.rs:212.)  A subset is a bitmap over the corpus's indices,
 * resident on the corpus's device.  Each subset call derives, in one pass over the tiles, slot metadata in which every
 * non-member is an unused slot, and runs the match pipeline of the full call through it.
 *
 * frz_match_list_subset(m, c, s) is bit-identical to [r for r in frz_match_list(m, c) if r.index is a member of s], in
 * the same order, for every matcher and sort strategy (per-haystack results do not depend on the other rows, and the
 * sorts are stable on (score, index)).  The empty matcher returns the live members in index order, reversed for the
 * *_DESC strategies.
 *
 * A subset belongs to the corpus it was made on: another corpus is FRZ_ERR_INVALID_ARG, and it must be destroyed before
 * that corpus.  The match calls only read it, so several matchers may use it at once.  Membership is by index and
 * survives edits of the corpus: rows appended after frz_subset_create are not members, a removed member stops matching
 * as everywhere else, a replaced member stays a member with its new text. */
typedef struct frz_subset frz_subset;
/* The set {which[0..n)} of indices of `c` (any order, duplicates allowed), resident on c's device.  An index >=
 * frz_corpus_len(c), or NULL with n > 0, is FRZ_ERR_INVALID_ARG; n == 0 is the empty set. */
FRZ_API frz_status frz_subset_create(const frz_corpus* c, const uint32_t* which, uint64_t n, frz_subset** out);
/* distinct indices given at creation, rows removed before or after it included (those never match, so the live count
 * can be lower) */
FRZ_API uint64_t frz_subset_len(const frz_subset* s);
FRZ_API void frz_subset_destroy(frz_subset* s);
/* frz_match_list restricted to the members: same arguments and capacity rule (FRZ_ERR_CAPACITY, *n_out = needed; room
 * for frz_subset_len(s) matches suffices) */
FRZ_API frz_status frz_match_list_subset(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s,
                                         frz_match* out, uint64_t cap, uint64_t* n_out);
/* frz_match_list_top restricted to the members: same rules as frz_match_list_top.  The first min(k, total) rows of
 * frz_match_list_subset's list; *n_total = its length.  Room for min(k, frz_subset_len(s)) matches in `out` suffices. */
FRZ_API frz_status frz_match_list_subset_top(frz_matcher* m, const frz_corpus* corpus, const frz_subset* s, uint64_t k,
                                             frz_match* out, uint64_t* n_out, uint64_t* n_total);

/* ---------------------------------------------------------------- subsets from attributes
 *
 * A filter on structured fields of the rows that changes with every request: a shell history searched "from the last 7
 * days, exit status != 0, on this host", a file picker searched "*.rs or *.toml, modified since yesterday", a launcher
 * searched "in these three categories".  The reference has no such method: its callers filter the haystacks themselves
 * before Matcher::match_list (src/matcher/mod.rs:212).  Here the fields stay resident beside the corpus as attribute
 * handles, and frz_subset_where fills an ordinary subset from a conjunction of clauses over them on the device, so every
 * call that takes a subset (the subset, ranked, collapsed, column and batched calls) filters without any change.
 *
 * An attribute is a signed 64-bit value per index of a corpus, resident on the corpus's device; FRZ_ATTR_NULL, and every
 * index without a value, is "no value", which never satisfies a clause, negated or not.  It follows frz_boost's rules: it
 * belongs to the corpus it was made on (another corpus is FRZ_ERR_INVALID_ARG, and it must be destroyed before that
 * corpus), and values are kept by index across corpus edits: a removed row keeps its value, a replaced row keeps its
 * value, and rows appended after frz_attr_create are null until frz_attr_set gives them a value.
 *
 * To filter per request, create an empty subset once (frz_subset_create(c, NULL, 0, &s)) and refill it with
 * frz_subset_where: its device buffers only grow, so steady-state requests allocate nothing. */
#define FRZ_ATTR_NULL INT64_MIN          /* "no value": never satisfies a clause, negated or not */
#define FRZ_WHERE_MAX_CLAUSES 8
#define FRZ_WHERE_MAX_IN 4096            /* set values over all clauses of one call */
typedef struct frz_attr frz_attr;
/* The reference has no such method (see above).  values[i] is the value of index i for i < n; the others are null.
 * n > frz_corpus_len(c), or NULL values with n > 0, is FRZ_ERR_INVALID_ARG; n == 0 is an all-null attribute. */
FRZ_API frz_status frz_attr_create(const frz_corpus* c, const int64_t* values, uint64_t n, frz_attr** out);
/* The reference has no such method (see above).  value[which[j]] = values[j] for j < n (FRZ_ATTR_NULL clears a value).
 * An index >= frz_corpus_len(c) at the time of the call (rows appended since creation may be set), a duplicate index, or
 * NULL arrays with n > 0 is FRZ_ERR_INVALID_ARG; every argument is checked before anything changes, so a refused call
 * leaves the attribute as it was.  n == 0 does nothing.  Synchronous; it must not run concurrently with a
 * frz_subset_where reading a. */
FRZ_API frz_status frz_attr_set(frz_attr* a, const uint32_t* which, const int64_t* values, uint64_t n);
FRZ_API void frz_attr_destroy(frz_attr* a);
/* The reference has no such method (see above).  out[i] = value[i] for i < n (FRZ_ATTR_NULL where there is none), e.g.
 * the ranks frz_attr_rank wrote.  n > frz_corpus_len(c), or NULL out with n > 0, is FRZ_ERR_INVALID_ARG.  Synchronous. */
FRZ_API frz_status frz_attr_get(const frz_attr* a, int64_t* out, uint64_t n);

/* One clause of frz_subset_where over v, an index's value in `attr`. */
typedef struct frz_where_clause {
    const frz_attr* attr;
    int64_t lo, hi;          /* range clause (n_in == 0): lo <= v <= hi  (lo > hi: holds for no value) */
    const int64_t* in;       /* set clause (n_in > 0): v is one of in[0..n_in), any order, duplicates allowed */
    uint64_t n_in;
    int32_t negate;          /* nonzero: the clause holds where its test fails (still never for a null value) */
} frz_where_clause;

/* The reference has no such method (see above).  Replaces the contents of s, which keeps its corpus c: afterwards s holds
 * exactly the indices i < frz_corpus_len(c) that are members of `base` (when base is not NULL; indices at or beyond its
 * bitmap's length are not members) and for which every clause holds.  n_clauses == 0 selects every index, restricted to
 * base.  Removed rows are included as frz_subset_create includes them: frz_subset_len counts them and the match calls
 * skip them.  For every call that takes a subset, the filled s behaves bit for bit like frz_subset_create(c, <those
 * indices>).  base may be s itself (refining in place).  Synchronous: it returns after the member count is read back.  It
 * must not run concurrently with a call that reads s or base.
 *
 * Checked in this order before any device work, leaving s as it was: a NULL s, or NULL clauses with n_clauses > 0
 * (FRZ_ERR_INVALID_ARG); more than FRZ_WHERE_MAX_CLAUSES clauses (FRZ_ERR_UNSUPPORTED); a NULL attr, or NULL in with
 * n_in > 0 (FRZ_ERR_INVALID_ARG); more than FRZ_WHERE_MAX_IN set values in all (FRZ_ERR_UNSUPPORTED); a set value equal
 * to FRZ_ATTR_NULL (FRZ_ERR_INVALID_ARG); an attribute or base of another corpus (FRZ_ERR_INVALID_ARG).  A failure after
 * the checks (out of device memory, for example) leaves s as the empty set, never half-written. */
FRZ_API frz_status frz_subset_where(frz_subset* s, const frz_where_clause* clauses, uint64_t n_clauses, const frz_subset* base);
/* The reference has no such method (see above).  frz_subset_where for q subsets of one corpus in one call, as a server
 * answering many filtered requests at once needs before a batched match call: one upload, one pass over the attribute
 * values in which each chunk of rows is read once for every query, one read-back of the q member counts and one
 * synchronise.  Query j's clauses are clauses[o_j .. o_j + n_clauses[j]), o_j being the sum of the earlier n_clauses,
 * and its base is bases[j] (bases == NULL: no query has a base).  Afterwards each s[j] is bit for bit what
 * frz_subset_where(s[j], clauses + o_j, n_clauses[j], bases[j]) leaves, for every call that takes a subset.  Every s[j],
 * attribute and base belongs to s[0]'s corpus.  The s[j] are distinct; bases[j] may be s[j] itself (refining it in
 * place) or any subset that is not another query's s[i], and several queries may share a base.  The per-query limits
 * are frz_subset_where's (FRZ_WHERE_MAX_CLAUSES clauses, FRZ_WHERE_MAX_IN set values).  The subsets' device buffers and
 * the call's staging (kept on the corpus) only grow, so steady-state refills at the same q allocate nothing.  The call
 * runs its batched kernels from q = 2, except for q = 2 on a corpus of more than 2^22 rows; there, and for q = 1, it
 * runs frz_subset_where query by query, which measured faster (DESIGN.md §4.14, "Batched fills").  Synchronous; it must not run concurrently with a call that reads any s[j] or base, or with
 * another frz_subset_where_batch on the same corpus.
 *
 * Checked in this order before any device work, leaving every subset as it was: NULL s or n_clauses with q > 0
 * (FRZ_ERR_INVALID_ARG); query by query, frz_subset_where's checks in its order up to the corpus checks (a NULL s[j], or
 * NULL clauses with n_clauses[j] > 0, ...); query by query, an s[j], attribute or base of another corpus than s[0]'s
 * (FRZ_ERR_INVALID_ARG); an s[j] given twice (FRZ_ERR_INVALID_ARG); a bases[j] that is s[i] for some i != j
 * (FRZ_ERR_INVALID_ARG).  The message names the query.  q == 0 makes no CUDA call.  A failure after the checks (out of
 * device memory, for example) leaves every s[j] as the empty set. */
FRZ_API frz_status frz_subset_where_batch(frz_subset* const* s, uint64_t q, const frz_where_clause* clauses,
                                          const uint64_t* n_clauses, const frz_subset* const* bases);

/* ---------------------------------------------------------------- subsets from text queries
 *
 * A scope on the rows' text that changes with every request: a file picker searched "under src/", "only *.rs" or "not in
 * node_modules", a shell history searched "commands run under this project".  The reference writes such scopes in its
 * own query syntax (Pattern::parse_query: ^prefix, suffix$, 'exact, !not, several atoms ANDed), and a haystack is in
 * Matcher::match_list exactly when the prefilter of every non-negated pattern accepts it and that of no negated pattern
 * does (src/matcher/algo.rs:85-100, src/matcher/multi.rs:84-152).  frz_subset_match fills an ordinary subset with those
 * rows on the device, from the prefilter stage alone: no scoring, sorting or copy-out. */

/* The reference has no such method (see above).  Let C be s's corpus and T be `text` (NULL: T = C).  Replaces the contents
 * of s, which keeps its corpus C: afterwards s holds exactly the indices i < frz_corpus_len(C) that are members of `base`
 * (when base is not NULL; indices at or beyond its bitmap's length are not members) and that are the index of a row of
 * frz_match_list_into(m, T, 0).  So T's row i is live, passes every non-negated compiled pattern's length gate and
 * prefilter and no negated pattern's; the empty matcher matches every live row, and an all-negated matcher every live row
 * that no pattern matches.  T may be another corpus with the same index space (a column of the same rows, as the text
 * keys of frz_attr_rank may be): for example a subset of a file-name corpus filled from a query over the directory
 * corpus.  For every call that takes a subset, the filled s behaves bit for bit like frz_subset_create(C, <those
 * indices>), and frz_subset_len is their number.  base may be s itself (refining in place).  Synchronous: it returns
 * after the member count is read back, with one read-back and one synchronise.  It must not run concurrently with another
 * call on m, or with a call that reads s or base.  s's device buffers only grow, and so does m's workspace, which the
 * fill uses as a match call does, so a steady-state refill allocates nothing.
 *
 * Checked in this order before any device work, leaving s as it was: a NULL s or m (FRZ_ERR_INVALID_ARG); T on another
 * device than C, or with another frz_corpus_len (FRZ_ERR_INVALID_ARG); a base of another corpus than C
 * (FRZ_ERR_INVALID_ARG); more rows than u32 indices reach (FRZ_ERR_TOO_MANY_ITEMS); no usable device (FRZ_ERR_NO_DEVICE:
 * there is no CPU fallback).  A failure after the checks (out of device memory, for example) leaves s as the empty set. */
FRZ_API frz_status frz_subset_match(frz_subset* s, frz_matcher* m, const frz_corpus* text, const frz_subset* base);
/* Test aid: force 1 makes this thread's frz_subset_match prefilter every pattern after the first, and the first one when a
 * base is given, through slot metadata masked to the members so far; force 2 never does; force 0 restores its rule (the
 * masked form for every pattern after the first, and for the first when the base leaves rows out, DESIGN.md §4.19);
 * force < 0 changes nothing.  Returns how many patterns this thread's last frz_subset_match prefiltered through masked
 * metadata. */
FRZ_API uint32_t frz_debug_subset_match(int force);

/* Ranks from several keys.  An order by name, or by a key and then a name, needs a key the caller does not hold: the
 * dense rank of each row's text.  frz_attr_rank fills an attribute on the device with each row's place in a lexicographic
 * order of up to FRZ_RANK_MAX_KEYS keys, each an attribute or the text of a corpus, so that every call that takes an
 * attribute (the ordered calls, frz_subset_where) orders or filters by it unchanged. */
#define FRZ_RANK_MAX_KEYS 4
typedef struct frz_rank_key {
    const frz_attr* attr;      /* an attribute key, or NULL */
    const frz_corpus* text;    /* a text key: the haystacks of this corpus, or NULL; exactly one of attr / text */
    uint32_t desc;             /* nonzero: larger values / later texts first */
    uint32_t fold_case;        /* text keys only: ASCII A-Z compare as a-z */
} frz_rank_key;
/* The reference has no such method (see above).  Let C be a's corpus.  Row i < frz_corpus_len(C) is ranked when it is live
 * in C and in the corpus of every text key (a removed row has no text).  Afterwards value[i] of a ranked row is the number
 * of distinct key tuples of ranked rows that come strictly before its own (a dense rank from 0: equal tuples share a
 * rank), and FRZ_ATTR_NULL for every other row.  Tuples compare key by key: an attribute key by value, reversed by desc,
 * a null value after every value in both directions; a text key by its bytes as unsigned bytes, a proper prefix first
 * (memcmp order: code point order for UTF-8), A-Z as a-z under fold_case, reversed by desc.  The values are a snapshot:
 * rows appended later are null until the next call, and edits of a key do not update them.  a may be one of the keys.
 * Synchronous; it must not run concurrently with a call that reads a or a key.
 *
 * Checked in this order before any device work, leaving a as it was: a NULL a, or NULL keys with n_keys > 0
 * (FRZ_ERR_INVALID_ARG); n_keys == 0 (FRZ_ERR_INVALID_ARG); more than FRZ_RANK_MAX_KEYS keys (FRZ_ERR_UNSUPPORTED); a key
 * with both or neither of attr and text (FRZ_ERR_INVALID_ARG); fold_case on an attribute key (FRZ_ERR_INVALID_ARG); a key
 * whose corpus is on another device or holds another number of rows than C (FRZ_ERR_INVALID_ARG).  A failure after the
 * checks (out of device memory, for example) leaves a's values as they were.  Scratch stays on a and only grows, so a
 * refill at the same size allocates nothing. */
FRZ_API frz_status frz_attr_rank(frz_attr* a, const frz_rank_key* keys, uint64_t n_keys);

/* ---------------------------------------------------------------- ranked calls
 *
 * Completion menus, history searches and file pickers rank rows by the fuzzy score plus a per-row prior (frecency,
 * recency, pinned items).  The reference has no such method: its callers re-rank Matcher::match_list's output
 * (src/matcher/mod.rs:212-222) themselves.  These calls replace that re-rank and return only the first k rows.
 *
 * A boost is a signed 16-bit value per index of a corpus, resident on the corpus's device; indices without a value have
 * boost 0.  A row's key is clamp(score + boost[index], 0, 65535), computed in 32-bit arithmetic.
 * frz_match_list_ranked(m, c, s, b, k) takes the rows of frz_match_list_into(m, c, 0) (restricted to the members of s
 * as frz_match_list_subset does), reverses them under IndexDesc / ScoreThenIndexDesc, sorts them stably by descending
 * key, and returns the first min(k, total) rows.  The rows are those of frz_match_list, bit for bit; only their order
 * differs.  Equal keys keep index order (ascending, or descending for the *_DESC strategies); raw scores do not break
 * ties.  Every strategy ranks by key, and the empty matcher ranks too: it lists the live rows by descending boost.  With
 * an all-zero boost under ScoreThenIndexAsc / Desc the result equals frz_match_list_top(m, c, k).
 *
 * A boost belongs to the corpus it was made on: another corpus is FRZ_ERR_INVALID_ARG, and it must be destroyed before
 * that corpus.  Ranked calls only read it, so several matchers may share one.  Boosts are kept by index across corpus
 * edits: a removed row stops matching, a replaced row keeps its boost, and rows appended after frz_boost_create have
 * boost 0 until frz_boost_set gives them one. */
typedef struct frz_boost frz_boost;
/* The reference has no such method (see above).  values[i] is the boost of index i for i < n; the others are 0.
 * n > frz_corpus_len(c), or NULL values with n > 0, is FRZ_ERR_INVALID_ARG; n == 0 is an all-zero boost. */
FRZ_API frz_status frz_boost_create(const frz_corpus* c, const int16_t* values, uint64_t n, frz_boost** out);
/* The reference has no such method (see above).  boost[which[j]] = values[j] for j < n.  An index >=
 * frz_corpus_len(c) at the time of the call (rows appended since creation may be set), a duplicate index, or NULL arrays
 * with n > 0 is FRZ_ERR_INVALID_ARG; every argument is checked before anything changes, so a refused call leaves the
 * boost as it was.  n == 0 does nothing.  Synchronous; it must not run concurrently with a ranked call reading b. */
FRZ_API frz_status frz_boost_set(frz_boost* b, const uint32_t* which, const int16_t* values, uint64_t n);
FRZ_API void frz_boost_destroy(frz_boost* b);
/* The reference has no such method (see above).  out[i] = boost[i] for i < n (0 where there is none).
 * n > frz_corpus_len(c), or NULL out with n > 0, is FRZ_ERR_INVALID_ARG.  Synchronous. */
FRZ_API frz_status frz_boost_get(const frz_boost* b, int16_t* out, uint64_t n);

/* Boosts from attribute rules.  Most priors are relative to the request: "modified in the last hour +30, last day +20",
 * "in the caller's directory +15", "pinned +50".  frz_boost_where fills a boost on the device from rules over the
 * resident attributes (frz_attr), each a frz_subset_where clause and the amount it adds, so a ranked call's boost follows
 * every request without a host pass over the rows or an upload of their values.  A rule whose add is a function of the
 * value (a linear decay) is a ladder of range rules. */
#define FRZ_BOOST_MAX_RULES 8
typedef struct frz_boost_rule {
    frz_where_clause when;   /* the rule applies to an index for which this clause holds (a null value: never, negated or not) */
    int32_t add;             /* -65535 .. 65535 */
} frz_boost_rule;
/* The reference has no such method (see above).  Let C be b's corpus.  Afterwards, for every index i < frz_corpus_len(C),
 * removed rows included (boosts are kept by index), boost[i] = clamp(base_i + the sum of the adds of the rules whose clause
 * holds for i, -32768, 32767), the sum in 32-bit arithmetic (it cannot overflow); base_i is base's boost of i, 0 when base
 * is NULL.  A clause means what it means in frz_subset_where (range or set, negation, a null value never holds).  base may
 * be b itself (adding to it in place); n_rules == 0 copies base, or zeroes b without one.  Rows appended later have
 * boost 0 until the next fill or frz_boost_set, which works on a filled boost as on any other.  b's key bound, which
 * the ranked calls add to the score bound, becomes max(0, the largest value filled), reduced on the device and read
 * back exactly.  Synchronous: it returns after that read-back, the call's one synchronise.  It must not run concurrently
 * with a call that reads b or base.  Its device scratch (the uploaded rules, set values and maxima) stays on b and only
 * grows, and b's values grow once to C's length, so a steady-state refill allocates nothing.
 *
 * Checked in this order before any device work, leaving b as it was: a NULL b, or NULL rules with n_rules > 0
 * (FRZ_ERR_INVALID_ARG); more than FRZ_BOOST_MAX_RULES rules (FRZ_ERR_UNSUPPORTED); a rule with a NULL attr, or NULL in
 * with n_in > 0 (FRZ_ERR_INVALID_ARG); a rule's add outside -65535 .. 65535 (FRZ_ERR_INVALID_ARG); more than
 * FRZ_WHERE_MAX_IN set values in all (FRZ_ERR_UNSUPPORTED); a set value equal to FRZ_ATTR_NULL (FRZ_ERR_INVALID_ARG); an
 * attribute or base of another corpus (FRZ_ERR_INVALID_ARG).  The message names the rule.  Out of device memory while
 * growing b's values leaves b as it was.  A CUDA failure after that leaves b's values unspecified and its key bound at
 * 32767, which still bounds every value. */
FRZ_API frz_status frz_boost_where(frz_boost* b, const frz_boost_rule* rules, uint64_t n_rules, const frz_boost* base);
/* The reference has no such method (see above).  frz_boost_where for q boosts of one corpus in one call, as a server
 * answering many users' "my directory and my recent rows first" requests needs before frz_match_list_batch: one upload,
 * one pass in which each chunk of each distinct attribute is read once for every query, one read-back of the q key
 * bounds and one synchronise.  Query j's rules are rules[o_j .. o_j + n_rules[j]), o_j being the sum of the earlier
 * n_rules, and its base is bases[j] (bases == NULL: no query has a base).  Afterwards each b[j] holds, bit for bit, the
 * values and key bound that frz_boost_where(b[j], rules + o_j, n_rules[j], bases[j]) leaves.  Every b[j], attribute and
 * base belongs to b[0]'s corpus.  The b[j] are distinct; bases[j] may be b[j] itself or any boost that is not another
 * query's b[i], and several queries may share a base.  The per-query limits are frz_boost_where's.  The call's scratch
 * stays on b[0] and only grows.  Synchronous; it must not run concurrently with a call that reads any b[j] or base.
 *
 * Checked in this order before any device work, leaving every boost as it was: NULL b or n_rules with q > 0
 * (FRZ_ERR_INVALID_ARG); query by query, frz_boost_where's checks in its order up to the corpus checks; query by query, a
 * b[j], attribute or base of another corpus than b[0]'s (FRZ_ERR_INVALID_ARG); a b[j] given twice (FRZ_ERR_INVALID_ARG);
 * a bases[j] that is b[i] for some i != j (FRZ_ERR_INVALID_ARG).  The message names the query.  q == 0 makes no CUDA
 * call.  Failures after the checks leave each b[j] as frz_boost_where's would. */
FRZ_API frz_status frz_boost_where_batch(frz_boost* const* b, uint64_t q, const frz_boost_rule* rules, const uint64_t* n_rules,
                                         const frz_boost* const* bases);
/* The reference has no such method (see above).  The first min(k, total) rows ranked by key; *n_total = total (may be
 * NULL).  s: NULL for the whole corpus, or a subset of the same corpus.  Same rules as frz_match_list_top: `out` is HOST
 * memory with room for k matches (min(k, frz_corpus_len(c)) suffices, or min(k, frz_subset_len(s)) with a subset),
 * k = 0 only counts, k = UINT64_MAX ranks the whole list, a NULL `out` with k > 0 is FRZ_ERR_INVALID_ARG, and the call
 * never returns FRZ_ERR_CAPACITY.  A NULL matcher, corpus or boost, or a boost or subset of another corpus, is
 * FRZ_ERR_INVALID_ARG. */
FRZ_API frz_status frz_match_list_ranked(frz_matcher* m, const frz_corpus* c, const frz_subset* s, const frz_boost* b,
                                         uint64_t k, frz_match* out, uint64_t* n_out, uint64_t* n_total);

/* ---------------------------------------------------------------- ordered calls
 *
 * A shell history lists the most recent matching command first, a log or mail search sorts "newest first", a file picker
 * sorts by "last modified", and a completion menu breaks score ties by a precomputed sort key.  The reference has no such
 * method: its callers sort Matcher::match_list's output (src/matcher/mod.rs:212-222) by their own copy of the field.  These
 * calls order the matches by an attribute (frz_attr above) on the device and return only the first k rows. */
enum {
    FRZ_ORDER_ATTR_DESC = 0,              /* by value, largest first (newest first) */
    FRZ_ORDER_ATTR_ASC = 1,               /* by value, smallest first */
    FRZ_ORDER_SCORE_THEN_ATTR_DESC = 2,   /* by score (with the boost), then by value, largest first */
    FRZ_ORDER_SCORE_THEN_ATTR_ASC = 3     /* by score (with the boost), then by value, smallest first */
};
/* The reference has no such method (see above).  Let L0 be the rows of frz_match_list_into(m, c, 0), restricted to the
 * members of s when s is given (as frz_match_list_subset does), and reversed under IndexDesc / ScoreThenIndexDesc.  Let
 * v(i) be index i's value in a; it is null when it equals FRZ_ATTR_NULL or when i lies past the attribute's values.  Let
 * r(i) be clamp(score + boost[i], 0, 65535) (32-bit arithmetic, frz_match_list_ranked's key) when b is given, else the
 * raw score.  L0 is sorted stably by:
 *   FRZ_ORDER_ATTR_DESC:             non-null rows first, then v descending, then r descending;
 *   FRZ_ORDER_ATTR_ASC:              non-null rows first, then v ascending, then r descending;
 *   FRZ_ORDER_SCORE_THEN_ATTR_DESC:  r descending, then non-null rows first, then v descending;
 *   FRZ_ORDER_SCORE_THEN_ATTR_ASC:   r descending, then non-null rows first, then v ascending.
 * Rows still tied keep L0's order: index order in the strategy's direction.  Nulls go last in both directions.  Every
 * strategy orders this way, and so does the empty matcher: it lists the live rows by the attribute ("latest first").  The
 * rows are those of frz_match_list, bit for bit, raw scores included; only their order differs.  The call writes the first
 * min(k, total) rows to `out`, their number to *n_out and total to *n_total (may be NULL).
 *
 * Same rules as frz_match_list_ranked: `out` is HOST memory with room for k matches (min(k, frz_corpus_len(c)) suffices,
 * or min(k, frz_subset_len(s)) with a subset), k = 0 only counts, k = UINT64_MAX returns the whole ordered list, and the
 * call never returns FRZ_ERR_CAPACITY.  Checked before any device work: a NULL matcher, corpus or attribute, or a NULL out
 * with k > 0, an order above FRZ_ORDER_SCORE_THEN_ATTR_ASC, or a subset, boost or attribute of another corpus is
 * FRZ_ERR_INVALID_ARG.  s and b may be NULL.  Blocking; it only reads its handles, so several matchers may share them. */
FRZ_API frz_status frz_match_list_ordered(frz_matcher* m, const frz_corpus* c, const frz_subset* s, const frz_boost* b,
                                          const frz_attr* a, uint32_t order, uint64_t k, frz_match* out, uint64_t* n_out,
                                          uint64_t* n_total);

/* ------------------------------------------------ collapsed calls: groups
 *
 * Rows that belong together (every execution of one command in a shell history, every hit of one file in a live grep,
 * every item of one section of a launcher) collapsed to their best rows on the device, with a match count per group.  The
 * reference has no such method: its caller de-duplicates or buckets Matcher::match_list's output itself
 * (src/matcher/mod.rs:212-222), which here means fetching the whole list.
 *
 * A group handle gives each corpus index a group id below n_groups, or FRZ_GROUP_NONE.  It follows frz_boost's rules: it
 * belongs to the corpus it was made on (another corpus is FRZ_ERR_INVALID_ARG, and it must be destroyed before that
 * corpus), calls only read it, so several matchers may share one, and ids are kept by index across corpus edits: a
 * removed row stops matching, a replaced row keeps its group, and rows appended after frz_groups_create are in no group
 * until frz_groups_set gives them one. */
#define FRZ_GROUP_NONE 0xFFFFFFFFu
typedef struct frz_groups frz_groups;
/* ids[i] is the group of index i for i < n; every other index is in no group.  n > frz_corpus_len(c), n_groups outside
 * 1 .. 2^32 - 1, an id >= n_groups other than FRZ_GROUP_NONE, or NULL ids with n > 0 is FRZ_ERR_INVALID_ARG. */
FRZ_API frz_status frz_groups_create(const frz_corpus* c, const uint32_t* ids, uint64_t n, uint64_t n_groups, frz_groups** out);
/* group[which[j]] = ids[j] for j < n.  An index >= frz_corpus_len(c) at the time of the call (rows appended since creation
 * may be set), a duplicate index, an id >= n_groups other than FRZ_GROUP_NONE, or NULL arrays with n > 0 is
 * FRZ_ERR_INVALID_ARG; every argument is checked before anything changes.  n == 0 does nothing.  Synchronous; it must not
 * run concurrently with a call reading g. */
FRZ_API frz_status frz_groups_set(frz_groups* g, const uint32_t* which, const uint32_t* ids, uint64_t n);
FRZ_API uint64_t frz_groups_count(const frz_groups* g);   /* n_groups (0 for NULL) */
FRZ_API void frz_groups_destroy(frz_groups* g);
/* Let L be the list frz_match_list_ranked(m, c, s, b, UINT64_MAX) returns when b is given, else frz_match_list_subset(m,
 * c, s) when s is given, else frz_match_list(m, c).  Let C be the rows of L, in L's order, that are in no group or that
 * have fewer than per_group earlier rows of L in their group.  The call writes C[0 : min(k, |C|)] to `out`, bit for bit,
 * their number to *n_out and |C| to *n_total (may be NULL).  group_counts (may be NULL) is a host array of n_groups
 * entries: entry j receives the rows of L in group j, counted before collapsing.
 * per_group: 1 .. 32, or UINT64_MAX for no cap (C = L: the uncollapsed call plus the counts).  0 is FRZ_ERR_INVALID_ARG,
 * any other value FRZ_ERR_UNSUPPORTED.  The other rules are frz_match_list_ranked's: k = 0 only counts, k = UINT64_MAX
 * returns all of C, the call never returns FRZ_ERR_CAPACITY, and a NULL out with k > 0, a NULL matcher, corpus or groups,
 * or a subset, boost or groups handle of another corpus is FRZ_ERR_INVALID_ARG, checked before any device work.
 * Blocking. */
FRZ_API frz_status frz_match_list_collapsed(frz_matcher* m, const frz_corpus* c, const frz_subset* s, const frz_boost* b,
                                            const frz_groups* g, uint64_t per_group, uint64_t k, frz_match* out,
                                            uint64_t* n_out, uint64_t* n_total, uint32_t* group_counts);

/* ------------------------------------------------ column calls
 *
 * Rows with several text fields, each searched by its own query (file name + directory, command + working directory,
 * symbol + container, title + artist): a matcher per column, rows must match every column, scores add up.  The reference
 * has no such method; it is its multi-pattern rule (src/matcher/multi.rs:83-152) where each pattern reads its own column.
 *
 * Column c is the corpus cols[c], searched by ms[c].  All columns share one index space: row i is haystack i of every
 * column, and n is their common frz_corpus_len.  Let L_c be the rows of frz_match_list_into(ms[c], cols[c], 0) (an empty
 * matcher, or one whose patterns are all negated, lists every row it does not exclude, with score 0).  Row i matches
 * when i < n, it is live (not removed) in every column, it is a member of s when s is given, and it is in every L_c.  Its
 * record is index i, score min(65535, sum_c score_c(i)) and exact OR_c exact_c(i).  The list L: the matching rows in
 * index order, reversed under the *_DESC strategies, then
 *   b given:                                    ranked by key exactly as frz_match_list_ranked (every strategy);
 *   else some matcher has a compiled pattern
 *        and sort is ScoreThenIndexAsc / Desc:  sorted stably by descending score (src/matcher/mod.rs:218);
 *   else:                                       left in that order.
 * g given: C is L collapsed exactly as frz_match_list_collapsed collapses its L, and group_counts (may be NULL; a host
 * array of frz_groups_count(g) entries) receives L's rows per group.  Otherwise C = L.  The call writes C[0 : min(k, |C|)]
 * to `out` (HOST memory; min(k, frz_corpus_len, frz_subset_len(s)) entries suffice), their number to *n_out and |C| to
 * *n_total (may be NULL).  k = 0 only counts, k = UINT64_MAX returns all of C, and the call never returns
 * FRZ_ERR_CAPACITY.  per_group is read only when g is given: 1 .. 32 or UINT64_MAX; 0 is FRZ_ERR_INVALID_ARG, any other
 * value FRZ_ERR_UNSUPPORTED.  sort is an FRZ_SORT_* value; the matchers' own sort settings are not read.
 *
 * The order of the columns does not change the result (saturating addition of non-negative scores is associative, and
 * OR commutes), only the speed: the first column with a non-negated pattern is scanned in full, and every later pattern
 * runs on the rows that are still candidates, about 7 to 10 times slower per row than the full scan (DESIGN.md §4.9,
 * §4.13).  Put the most selective column first.  Every call, even with one column and one pattern, takes the
 * multi-pattern path: ms[0]'s device scratch grows by two candidate lists of 8 bytes per row (about 160 MB at 10 M rows,
 * kept for later calls), and a by-score sort does not get the histogram the single-pattern calls build while scoring.
 *
 * FRZ_ERR_INVALID_ARG, checked in this order before any device work: n_cols == 0; a NULL ms, cols, ms[c] or cols[c];
 * columns on different devices; columns whose frz_corpus_len differ at the time of the call (after an append to some
 * columns only, until the others catch up); then FRZ_ERR_TOO_MANY_ITEMS for more rows than u32 indices reach; then
 * FRZ_ERR_INVALID_ARG for a sort above 3; per_group 0 with groups (then FRZ_ERR_UNSUPPORTED for a
 * per_group out of range); a NULL out with k > 0; a subset, boost or groups handle made on none of the given columns.
 * Membership, boosts and group ids are by index, so a handle of any column serves.
 *
 * A column or a matcher may appear more than once.  Blocking.  The call runs on ms[0]'s device scratch and stream, and
 * frz_matcher_last_timings(ms[0]) reports it; the other matchers are only read, apart from their long-needle table, which
 * is uploaded to the columns' device.  None of the matchers, columns or handles may be used by another call meanwhile. */
FRZ_API frz_status frz_match_list_columns(frz_matcher* const* ms, const frz_corpus* const* cols, uint64_t n_cols,
                                          uint8_t sort, const frz_subset* s, const frz_boost* b, const frz_groups* g,
                                          uint64_t per_group, uint64_t k, frz_match* out, uint64_t* n_out,
                                          uint64_t* n_total, uint32_t* group_counts);

/* ------------------------------------------------ ordered collapsed and ordered column calls
 *
 * The default screen of a shell-history search shows each distinct command once, newest first; a live grep lists the
 * files with hits, most recently modified first; a launcher shows one entry per app, last used first.  Each needs the
 * rows grouped and the groups represented by their first rows in an attribute's order, not by their best-scoring rows.
 * A file picker orders file name + directory matches by modification time.  The reference has no such method: its
 * callers fetch the whole list and collapse or sort it on the host.  These calls do it on the device. */

/* The reference has no such method (see above).  Let L be the list frz_match_list_ordered(m, c, s, b, a, order,
 * UINT64_MAX, ...) returns: the rows of frz_match_list_into restricted to the members of s, reversed under the *_DESC
 * strategies, sorted stably by the order key (with the boost inside r), nulls last, remaining ties in index order.  Let C
 * be the rows of L, in L's order, that are in no group or that have fewer than per_group earlier rows of L in their group
 * (frz_match_list_collapsed's rule applied to this L).  The call writes C[0 : min(k, |C|)] to `out`, bit for bit, their
 * number to *n_out and |C| to *n_total (may be NULL).  group_counts (may be NULL) is a host array of
 * frz_groups_count(g) entries: entry j receives the rows of L in group j, counted before collapsing.
 * per_group: 1 .. 32, or UINT64_MAX for no cap (C = L: frz_match_list_ordered plus the counts).  With the empty matcher
 * the call lists the live rows, so per_group = 1 and FRZ_ORDER_ATTR_DESC over a timestamp gives the latest row of each
 * group, newest first.
 *
 * Every other rule is frz_match_list_ordered's: `out` is HOST memory with room for k matches (min(k, frz_corpus_len(c))
 * suffices, or min(k, frz_subset_len(s)) with a subset), k = 0 only counts, k = UINT64_MAX returns all of C, and the call
 * never returns FRZ_ERR_CAPACITY.  Checked in this order before any device work: FRZ_ERR_INVALID_ARG for a NULL matcher,
 * corpus, attribute or groups; per_group 0 (then FRZ_ERR_UNSUPPORTED for any other per_group out of range); a NULL out
 * with k > 0; an order above FRZ_ORDER_SCORE_THEN_ATTR_ASC; a subset, boost, groups or attribute handle of another corpus
 * (the first one reported in that order).  s and b may be NULL.  Blocking; it only reads its handles. */
FRZ_API frz_status frz_match_list_ordered_collapsed(frz_matcher* m, const frz_corpus* c, const frz_subset* s,
                                                    const frz_boost* b, const frz_attr* a, uint32_t order,
                                                    const frz_groups* g, uint64_t per_group, uint64_t k, frz_match* out,
                                                    uint64_t* n_out, uint64_t* n_total, uint32_t* group_counts);

/* The reference has no such method (see above).  Let L0 be the joined rows of frz_match_list_columns(ms, cols, n_cols,
 * sort, s, ...) before its ordering step: the rows that match in every column, each with the saturating sum of its
 * column scores and the OR of its exact flags, in index order, reversed under the *_DESC strategies of `sort`.  L is L0
 * ordered by the attribute exactly as frz_match_list_ordered orders its L0, with the boost inside r (r is the summed
 * score, clamped with the boost).  With g, C is L collapsed as frz_match_list_ordered_collapsed collapses its L and
 * group_counts (may be NULL) receives L's rows per group; without g, C = L and per_group and group_counts are not read.
 * The call writes C[0 : min(k, |C|)] to `out` (HOST memory), their number to *n_out and |C| to *n_total (may be NULL);
 * k = 0 only counts, k = UINT64_MAX returns all of C, never FRZ_ERR_CAPACITY.
 *
 * Checked in this order before any device work: frz_match_list_columns' column checks (n_cols, NULL matchers or
 * columns, devices, lengths, the index range, sort); then FRZ_ERR_INVALID_ARG for a NULL attribute; with g, per_group 0
 * (then FRZ_ERR_UNSUPPORTED for any other per_group out of range); a NULL out with k > 0; an order above
 * FRZ_ORDER_SCORE_THEN_ATTR_ASC; a subset, boost, groups or attribute handle made on none of the columns.  A handle of
 * any column serves every column.  Every other rule (scratch, speed, column order, sharing) is frz_match_list_columns'. */
FRZ_API frz_status frz_match_list_columns_ordered(frz_matcher* const* ms, const frz_corpus* const* cols, uint64_t n_cols,
                                                  uint8_t sort, const frz_subset* s, const frz_boost* b, const frz_attr* a,
                                                  uint32_t order, const frz_groups* g, uint64_t per_group, uint64_t k,
                                                  frz_match* out, uint64_t* n_out, uint64_t* n_total,
                                                  uint32_t* group_counts);

/* frz_match_list_batch_top (above) where each query may have its own subset and boost, in one call: a service whose users
 * each search their own rows (a subset) ranked by a prior (a boost).  The reference has no such method (see the subset
 * and ranked calls above).  For every j < q, out[j*k .. j*k + n_out[j]), n_out[j] and n_total[j] are bit for bit what the
 * matching single-query call returns, for every matcher, config and sort strategy:
 *   boosts[j] != NULL:       frz_match_list_ranked(ms[j], corpus, subsets[j], boosts[j], k, ...);
 *   else subsets[j] != NULL: frz_match_list_subset_top(ms[j], corpus, subsets[j], k, ...);
 *   else:                    frz_match_list_top(ms[j], corpus, k, ...).
 * subsets and boosts may be NULL, meaning every entry is NULL; frz_match_list_batch(ms, q, c, NULL, NULL, k, ...) is
 * frz_match_list_batch_top(ms, q, c, k, ...).  All other argument rules, the batched class and its limits are
 * frz_match_list_batch_top's.  A subset or boost made on another corpus is FRZ_ERR_INVALID_ARG; every argument is checked
 * before any device work.  The same subset, boost or matcher may appear for many queries; the call only reads them.
 * A batched-class query runs the batched kernels whether or not it is scoped or ranked: its non-members are scored with
 * the rest of the corpus and dropped when its rows are chosen (DESIGN.md §4.11). */
FRZ_API frz_status frz_match_list_batch(frz_matcher* const* ms, uint64_t q, const frz_corpus* corpus,
                                        const frz_subset* const* subsets, const frz_boost* const* boosts, uint64_t k,
                                        frz_match* out, uint64_t* n_out, uint64_t* n_total);

/* frz_match_list_batch (above) where each query may also collapse its rows by its own groups, in one call: a service that
 * shows each of its users their distinct commands, their best hits per file or their section sizes.  For every j < q,
 * out[j*k .. j*k + n_out[j]), n_out[j], n_total[j] and, when given, group_counts[j] are bit for bit what the matching
 * single-query call returns:
 *   groups[j] != NULL: frz_match_list_collapsed(ms[j], corpus, subsets[j], boosts[j], groups[j], per_group[j], k, ...,
 *                      group_counts[j]);
 *   else:              query j of frz_match_list_batch (ranked, subset-top or top).
 * groups, subsets, boosts and group_counts may be NULL, meaning every entry is NULL; group_counts[j] (NULL, or a host array
 * of frz_groups_count(groups[j]) entries) is read only for a query with groups.  per_group may be NULL, meaning 1 for every
 * query; every entry follows frz_match_list_collapsed's rule (1 .. 32 or UINT64_MAX; 0 is FRZ_ERR_INVALID_ARG, any other
 * value FRZ_ERR_UNSUPPORTED).  A groups handle made on another corpus is FRZ_ERR_INVALID_ARG.  Every other rule is
 * frz_match_list_batch's, and every argument is checked before any device work.  A batched-class query with groups runs
 * the batched kernels, except one whose groups hold more than about 22 M ids, or one that asks for the counts of more
 * than 2^18 groups: those run the single-query call inside the same call (DESIGN.md §4.11). */
FRZ_API frz_status frz_match_list_batch_collapsed(frz_matcher* const* ms, uint64_t q, const frz_corpus* corpus,
                                                  const frz_subset* const* subsets, const frz_boost* const* boosts,
                                                  const frz_groups* const* groups, const uint64_t* per_group, uint64_t k,
                                                  frz_match* out, uint64_t* n_out, uint64_t* n_total, uint32_t* const* group_counts);

/* frz_match_list_batch_collapsed (above) where each query may also order its rows by its own attribute, in one call: a
 * shared shell-history server showing each user their distinct commands newest first, or a mail service listing each
 * user's hits newest first.  For every j < q, out[j*k .. j*k + n_out[j]), n_out[j], n_total[j] and, when given,
 * group_counts[j] are bit for bit what the matching single-query call returns:
 *   attrs[j] and groups[j] != NULL: frz_match_list_ordered_collapsed(ms[j], corpus, subsets[j], boosts[j], attrs[j],
 *                                   orders[j], groups[j], per_group[j], k, ..., group_counts[j]);
 *   attrs[j] != NULL, no groups:    frz_match_list_ordered(ms[j], corpus, subsets[j], boosts[j], attrs[j], orders[j], k, ...);
 *   else:                           query j of frz_match_list_batch_collapsed.
 * attrs, subsets, boosts, groups and group_counts may be NULL, meaning every entry is NULL; orders may be NULL, meaning
 * FRZ_ORDER_ATTR_DESC for every query; per_group may be NULL, meaning 1 for every query.  Rows out[j*k + n_out[j] ..
 * (j+1)*k) are not written.  Never FRZ_ERR_CAPACITY.
 *
 * Checked in this order before any device work: FRZ_ERR_INVALID_ARG for a NULL ms or corpus, or a NULL ms[j]; every
 * per_group[j] as frz_match_list_batch_collapsed checks it; FRZ_ERR_INVALID_ARG for an orders[j] above
 * FRZ_ORDER_SCORE_THEN_ATTR_ASC (every entry is checked, with or without an attribute); a subset, boost, groups or
 * attribute handle of another corpus (query by query, in that order within a query); a NULL n_out with q > 0; q*k
 * overflowing uint64_t or size_t; a NULL out with q*k > 0.  q = 0 then returns FRZ_OK without any CUDA call.
 *
 * The batched class and its limits are frz_match_list_batch_collapsed's.  Ordered queries run in sub-batches of their own,
 * whose last stage orders each query's rows by its order key on the device (DESIGN.md §4.11 "Ordered queries"); an ordered
 * query whose keys and tables do not fit two to a sub-batch, and every query of a sub-batch whose survivor lists
 * overflowed, runs its single-query call inside the same call.  frz_match_list_batch_collapsed is this call with
 * attrs == NULL. */
FRZ_API frz_status frz_match_list_batch_ordered(frz_matcher* const* ms, uint64_t q, const frz_corpus* corpus,
                                                const frz_subset* const* subsets, const frz_boost* const* boosts,
                                                const frz_attr* const* attrs, const uint32_t* orders,
                                                const frz_groups* const* groups, const uint64_t* per_group, uint64_t k,
                                                frz_match* out, uint64_t* n_out, uint64_t* n_total,
                                                uint32_t* const* group_counts);

/* frz_match_list_columns (above) for q queries over the same columns in one call: a service answering many users'
 * multi-field searches (file name + directory, command + working directory) over one set of columns.  Query j's matchers
 * are ms[j*n_cols .. (j+1)*n_cols), matcher c searching cols[c].  For every j < q, out[j*k .. j*k + n_out[j]), n_out[j],
 * n_total[j] and, when given, group_counts[j] are bit for bit what frz_match_list_columns(ms + j*n_cols, cols, n_cols, sort,
 * subsets[j], boosts[j], groups[j], per_group[j], k, ..., group_counts[j]) returns; rows out[j*k + n_out[j] .. (j+1)*k)
 * are not written.  subsets, boosts, groups and group_counts may be NULL, meaning every entry is NULL; per_group may be
 * NULL, meaning 1 for every query (frz_match_list_batch_collapsed's conventions).  sort is one FRZ_SORT_* value for every
 * query; the matchers' own sort settings are not read.
 *
 * Checked in this order before any device work: FRZ_ERR_INVALID_ARG for n_cols == 0; a NULL ms or cols; a NULL cols[c];
 * q*n_cols overflowing uint64_t or size_t; a NULL ms[i] for i < q*n_cols; columns on different devices; columns whose
 * frz_corpus_len differ (after an append to some columns only); then FRZ_ERR_TOO_MANY_ITEMS for more rows than u32 indices
 * reach; then FRZ_ERR_INVALID_ARG for a sort above 3; per_group[j] 0 (then FRZ_ERR_UNSUPPORTED for a per_group[j] out of
 * 1 .. 32 other than UINT64_MAX; every entry is checked, with or without groups); a subset, boost or groups handle made on
 * none of the columns; a NULL n_out with q > 0; q*k overflowing uint64_t or size_t; a NULL out with q*k > 0.  q = 0 then
 * returns FRZ_OK without any CUDA call.  Never FRZ_ERR_CAPACITY.  A matcher or a column may appear more than once.
 * Blocking; none of the matchers, columns or handles may be used by another call meanwhile.
 *
 * A query runs the batched kernels when every column's matcher either has no compiled pattern or has one pattern that is
 * fuzzy, not negated, on the byte path and at most 64 bytes long; at least one column has a pattern; every pattern has
 * max_typos = 0; k <= 1024; there are at most 255 columns; the columns hold at most 2^18 rows; and the call has at least
 * 32 such queries (frz_debug_batch_limits moves the row and query limits, and lets queries with a typo budget batch too).
 * DESIGN.md §4.13 measured that rule: queries with a typo budget, and corpora of 1 M rows, lost to the loop there.  Each sub-batch scans every column once for
 * the queries with a pattern in it and joins the columns per row on the device (DESIGN.md §4.13).  Grouped queries
 * follow frz_match_list_batch_collapsed's rules.  Every other query, and every query of a sub-batch whose survivor lists
 * overflowed, runs frz_match_list_columns inside the same call. */
FRZ_API frz_status frz_match_list_batch_columns(frz_matcher* const* ms, uint64_t q, const frz_corpus* const* cols, uint64_t n_cols,
                                                uint8_t sort, const frz_subset* const* subsets, const frz_boost* const* boosts,
                                                const frz_groups* const* groups, const uint64_t* per_group, uint64_t k,
                                                frz_match* out, uint64_t* n_out, uint64_t* n_total, uint32_t* const* group_counts);

/* Specialized::match_list / Matcher::match_list_into (src/matcher/algo.rs:17-22,
 * src/matcher/mod.rs:373-392): matches appended in input (index-ascending) order,
 * indices offset by `index_offset`, no sort. */
FRZ_API frz_status frz_match_list_into(frz_matcher* m, const frz_corpus* corpus, uint32_t index_offset,
                               frz_match* out, uint64_t cap, uint64_t* n_out);

/* End-to-end convenience: Matcher::match_list on HOST Arrow buffers (pack + H2D + match + D2H
 * in one call; nothing stays resident). */
FRZ_API frz_status frz_match_list_host(frz_matcher* m, const uint8_t* bytes, const uint64_t* offsets,
                               uint64_t n, int device, frz_match* out, uint64_t cap, uint64_t* n_out);
/* same, for either Arrow offset width (4 or 8 bytes); H2D chunks overlap the pack kernels */
FRZ_API frz_status frz_match_list_host_arrow(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width,
                                     uint64_t n, int device, frz_match* out, uint64_t cap, uint64_t* n_out);

/* Matcher::match_list_indices (src/matcher/mod.rs:234-262) for CHOSEN haystacks — the rows a UI is about to display:
 * for haystack which[j] (corpus-relative index) writes its Match to out_matches[j] and the byte offsets of the
 * matched characters, in the reference's descending order, to out_indices[j * stride ...]; out_counts[j] = how many
 * the haystack has (UNtruncated: when it exceeds `stride` only the first `stride` offsets were stored — call again with
 * a larger stride), or UINT32_MAX when that haystack does not match.  Host pointers.  Multi-pattern matchers pool
 * the atoms' indices like match_one_indices_multi (src/matcher/multi.rs:56-79).  Like the reference's, not a tuned path. */
FRZ_API frz_status frz_match_indices(frz_matcher* m, const frz_corpus* corpus, const uint32_t* which, uint64_t n,
                             frz_match* out_matches, uint32_t* out_indices, uint32_t stride, uint32_t* out_counts);

/* ------------------------------------------------ multi-GPU: match_list_parallel
 *
 * Matcher::match_list_parallel (src/matcher/parallel.rs:18-89) with GPUs in place of worker threads: the haystack list
 * is sharded by contiguous index range (shard g = [g*ceil(N/G), ...), SURVEY.md §8(e)), every GPU runs the whole local
 * pipeline on its shard with its own clone of the matcher (parallel.rs:46) and leaves a locally ordered run in HBM
 * (parallel.rs:67-73), ONE ncclAllGather moves the runs (padded to the longest) over NVLink, every GPU merges them
 * (k_merge_matches_by, src/k_merge.rs:90-131) and copies ITS slice of the merged list to the host buffer, so the
 * device->host copy runs over all PCIe links in parallel.  The match counts (the Vec lengths the k-merge reads) travel
 * through a small pinned host block shared by the ranks, published by each GPU as soon as its prefilter has run —
 * no second collective, and the exchange overlaps the scoring kernels.
 *
 * NCCL is loaded at run time (dlopen "libnccl.so.2", so a process that already carries PyTorch's NCCL shares it);
 * a communicator over ONE GPU never touches NCCL. */
typedef struct frz_comm frz_comm;
#define FRZ_UNIQUE_ID_BYTES 128

/* Single-process form — what a Rust caller of match_list_parallel uses: one communicator over `n_gpus` devices of this
 * process (`devices` NULL = 0..n_gpus-1), ncclCommInitAll, one worker thread per GPU inside the library (the
 * std::thread::scope pool of parallel.rs:39-66). */
FRZ_API frz_status frz_comm_create_local(int n_gpus, const int* devices, frz_comm** out);
/* Multi-process form (one rank per process: torchrun, MPI): rank 0 gets an id, the host program ships those 128 bytes
 * to every rank, every rank joins.  Collective: all ranks must call frz_comm_create_rank. */
FRZ_API frz_status frz_comm_unique_id(uint8_t id[FRZ_UNIQUE_ID_BYTES]);
FRZ_API frz_status frz_comm_create_rank(const uint8_t id[FRZ_UNIQUE_ID_BYTES], int world, int rank, int device, frz_comm** out);
FRZ_API void frz_comm_destroy(frz_comm* c);
FRZ_API int frz_comm_world(const frz_comm* c);
FRZ_API int frz_comm_rank(const frz_comm* c);      /* rank of this process (multi-process form), 0 for the local form */
FRZ_API int frz_comm_device(const frz_comm* c, int local_index);
/* Host buffer every rank's GPU can write: pinned; in the multi-process form ONE shared-memory segment mapped and pinned
 * by every rank (collective: every rank calls it with the same size and gets its own mapping of the same memory). */
FRZ_API frz_status frz_comm_host_alloc(frz_comm* c, uint64_t bytes, void** out);
FRZ_API frz_status frz_comm_host_free(frz_comm* c, void* p);
/* host-side barrier over the ranks of the communicator (no-op for the local form) */
FRZ_API frz_status frz_comm_barrier(frz_comm* c);

/* Contiguous index-range shards of one host Arrow list, shard g resident on the communicator's g-th GPU (local form).
 * `shards_out` receives frz_comm_world(c) corpora (empty shards are valid). */
FRZ_API frz_status frz_corpus_create_sharded(const uint8_t* bytes, const void* offsets, int offset_width, uint64_t n,
                                     frz_comm* c, frz_corpus** shards_out);

/* Matcher::match_list_parallel (src/matcher/parallel.rs:18-89), local form: shards[g] lives on the communicator's g-th
 * GPU and covers the indices after shards[0..g).  Blocking; `out` is host memory (frz_comm_host_alloc memory lets all
 * GPUs copy concurrently; any other memory works).  On FRZ_ERR_CAPACITY *n_out = needed. */
FRZ_API frz_status frz_match_list_parallel(frz_matcher* m, const frz_corpus* const* shards, int n_shards, frz_comm* c,
                                   frz_match* out, uint64_t cap, uint64_t* n_out);
/* One rank of the multi-process form.  Collective: every rank calls it with its shard and the index of its first
 * haystack.  `out` must be the buffer returned by frz_comm_host_alloc (every rank writes its slice of the merged list
 * into the shared segment; on return the WHOLE list is there) — or NULL with cap 0 to skip the host copy.
 * *d_out (optional) receives this rank's device copy of the merged list, valid until the next call on `c`. */
FRZ_API frz_status frz_match_list_parallel_rank(frz_matcher* m, const frz_corpus* shard, uint32_t index_offset, frz_comm* c,
                                        frz_match* out, uint64_t cap, uint64_t* n_out, const frz_match** d_out);
/* same, end to end: this rank's shard arrives as HOST Arrow buffers (streamed H2D + pack, as frz_match_list_host_arrow) */
FRZ_API frz_status frz_match_list_parallel_rank_host(frz_matcher* m, const uint8_t* bytes, const void* offsets, int offset_width,
                                             uint64_t n, uint32_t index_offset, frz_comm* c, frz_match* out, uint64_t cap,
                                             uint64_t* n_out);
/* Matcher::match_list_parallel (src/matcher/parallel.rs:18-89) followed by truncation to its first k rows (the reference
 * has no such method), local form: bit-identical to frz_match_list_parallel(...)[0 : min(k, total)].  Same arguments as
 * frz_match_list_parallel, with `k` in place of `cap`: `out` is host memory with room for `k` matches (room for min(k, the
 * haystacks of all shards) suffices: no more rows can match).  *n_out = min(k, total),
 * *n_total = total (may be NULL); k = 0 is valid; never FRZ_ERR_CAPACITY; NULL `out` with k > 0 is FRZ_ERR_INVALID_ARG.
 * Every GPU sorts only its run's first k and the exchange moves only what lands in the first min(k, total) positions. */
FRZ_API frz_status frz_match_list_parallel_top(frz_matcher* m, const frz_corpus* const* shards, int n_shards, frz_comm* c,
                                       uint64_t k, frz_match* out, uint64_t* n_out, uint64_t* n_total);
/* The same for one rank of the multi-process form (collective, like frz_match_list_parallel_rank): `out` is the
 * frz_comm_host_alloc buffer with room for k matches (on return the first min(k, total) rows are there), or NULL to skip
 * the host copy.  *n_out = min(k, total), *n_total = total (may be NULL).  *d_out (optional) receives this rank's device
 * copy of the merged list, whose first min(k, total) entries are the result, valid until the next call on `c`. */
FRZ_API frz_status frz_match_list_parallel_rank_top(frz_matcher* m, const frz_corpus* shard, uint32_t index_offset, frz_comm* c,
                                            uint64_t k, frz_match* out, uint64_t* n_out, uint64_t* n_total,
                                            const frz_match** d_out);
/* How host-out calls move the matches on this communicator: 2 = P2P placement (every GPU stores its matches at their
 * merged positions in the peers' slice buffers over NVLink — peer access in the local form, cudaIpc in the multi-process
 * form — then every GPU copies its slice out), 1 = NCCL slice exchange (grouped ncclSend/ncclRecv); -1 for a NULL
 * communicator.  2 on more than one GPU; the first call downgrades it to 1 when peer memory cannot be mapped, and
 * FRZ_PARALLEL_EXCHANGE=slices (a test hook) starts at 1.  Any other non-empty value of that variable makes
 * frz_comm_create_local / frz_comm_create_rank fail with FRZ_ERR_INVALID_ARG.  Device-out calls, and host-out calls whose
 * score bound needs the two-pass sort, use ncclAllGather of whole runs + merge. */
FRZ_API int frz_comm_exchange_mode(const frz_comm* c);

/* Device timings (ms) of the last parallel call on local rank `local_index`: [0] local pipeline (prefilter, scoring,
 * sort) [1] all-gather + merge [2] device->host slice [3] total; and the matcher clone that ran it (for
 * frz_matcher_last_timings).  Blocks until that rank's stream is idle. */
FRZ_API frz_status frz_comm_last_timings(frz_comm* c, int local_index, float* ms4, const frz_matcher** clone);

/* Device-resident variant used by the multi-GPU path (Matcher::match_list_parallel,
 * src/matcher/parallel.rs:18-89): this rank's shard → a locally ordered run left in HBM.
 * `d_out` (cap matches) and `d_count` (one uint64) are device pointers; `stream` is a
 * cudaStream_t (NULL = default stream).  Asynchronous: returns after enqueueing. */
FRZ_API frz_status frz_match_shard_device(frz_matcher* m, const frz_corpus* shard, uint32_t index_offset,
                                  frz_match* d_out, uint64_t cap, uint64_t* d_count, void* stream);
/* The count of a shard call is known before its scores (it is the prefilter's survivor count): this makes
 * `stream` (a second cudaStream_t) wait only until d_count has been written, so the count exchange of
 * match_list_parallel (the `Vec` lengths the reference's k-merge reads, src/k_merge.rs:96-104) overlaps scoring. */
FRZ_API frz_status frz_matcher_wait_count(frz_matcher* m, void* stream);

/* k_merge_matches_by (src/k_merge.rs:90-131) on device: `d_runs` holds `n_runs` runs, run r at
 * d_runs + r*run_stride with run_counts_host[r] valid entries, each already ordered per `sort`.
 * `score_bound`: upper bound of the scores in the runs (frz_matcher_score_bound), 0 = unknown.
 * Writes the merged sequence to d_out (may not alias d_runs).  Asynchronous on `stream`.  Uses one grow-only scratch
 * per device for the life of the process: calls for the same device must not overlap (one stream, or serialise). */
FRZ_API frz_status frz_merge_runs_device(const frz_match* d_runs, uint64_t run_stride,
                                 const uint64_t* run_counts_host, int n_runs, uint8_t sort,
                                 uint32_t score_bound, frz_match* d_out, int device, void* stream);
/* Upper bound of any score this matcher can emit (sum over its non-negated patterns, saturating at
 * 65535); lets the device sort / merge use a single counting pass.  0 for an empty matcher. */
FRZ_API uint32_t frz_matcher_score_bound(const frz_matcher* m);

/* Test aid: copies the compiled device pattern (frizbee_b200/csrc/frz_device.cuh: FrzPatternDev) of pattern i; out_size
 * must equal its size.  Lets host builds of the kernel cores run with exactly the constants the GPU receives. */
FRZ_API frz_status frz_matcher_debug_pattern(const frz_matcher* m, size_t i, void* out, size_t out_size);
/* Test aid: copies the needle (frizbee_b200/csrc/unicode_path.cuh: FrzUNeedle) and scoring constants (FrzUScoring) that
 * pattern i hands to the unicode, literal and traceback kernels; un_size / usc_size must equal their sizes.  Lets host
 * builds of unicode_path.cuh and indices_path.cuh run with exactly the constants the GPU receives. */
FRZ_API frz_status frz_matcher_debug_unicode(const frz_matcher* m, size_t i, void* un, size_t un_size, void* usc, size_t usc_size);

/* Test aid: copies the packed image of a corpus (frizbee_b200/csrc/frz_device.cuh, DESIGN.md §3) to host buffers, in
 * this order: tile_base (u64 per tile), groups (FrzGroupDesc, 16 bytes per group), slot_meta (u32 per slot), slot_of
 * (u16 per slot), slot_sig (2 x u32 per slot) and the packed units [0, total units) (16 bytes each).  With all six
 * buffers NULL, writes their sizes in bytes to sizes[0..5]; otherwise all six are needed and sizes[i] must equal those
 * sizes exactly.  Lets tests check the layout that every constructor and frz_corpus_append produce. */
FRZ_API frz_status frz_corpus_debug_image(const frz_corpus* c, void* tile_base, void* groups, void* slot_meta, void* slot_of,
                                  void* slot_sig, void* units, uint64_t sizes[6]);

/* Test aid: bytes of device memory the library holds right now, over every device (corpora, matchers, communicators
 * and internal scratch).  Lets tests check that repeated calls and destroyed objects leave nothing behind. */
FRZ_API uint64_t frz_debug_device_bytes(void);
/* Test aid: the most bytes frz_debug_device_bytes has held since the last call with reset != 0 (which first sets the mark
 * to the current value): the peak device memory of the calls in between. */
FRZ_API uint64_t frz_debug_device_bytes_peak(int reset);

/* radix_sort_matches (src/sort.rs:6-40): stable, descending score; `matches` is host memory. */
FRZ_API frz_status frz_radix_sort_matches(frz_match* matches, uint64_t n, int device);

/* Per-stage device timings (ms) of the most recent frz_match_list* call on this matcher:
 * [0]=prefilter [1]=smith-waterman [2]=sort/emit [3]=total device; bytes = algorithmic bytes. */
FRZ_API frz_status frz_matcher_last_timings(const frz_matcher* m, float* ms4, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* FRZ_CUDA_H */
