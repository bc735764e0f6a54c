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
