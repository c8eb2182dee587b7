/*
 * mpb200.h — C ABI of libmpb200.so, the H100 (sm_90a) implementation of multiPrime's degenerate-primer
 * candidate scan.  Loaded from Python with ctypes (multiprime_b200/_lib.py); no torch / C++ types cross
 * this boundary: plain pointers, sizes and opaque handles only.
 *
 * The reference (joybio/multiPrime) has no in-process API — its boundary is "python scripts/<tool>.py
 * <flags>" (multiPrime.py:202-206 etc.).  Each entry point below therefore names the reference FUNCTION it
 * replaces (core = scripts/multiPrime-core_V20.py); multiprime_b200/core.py re-assembles them behind the
 * reference's CLI.  INTEGRATION.md shows the ctypes binding a maintainer would add to the reference.
 *
 * Conventions
 *   - every function returns 0 on success, a negative MPB_E* code on failure; mpb_last_error() gives the
 *     message of the last failure on the calling thread.  CUDA errors are mapped, never abort().
 *   - "hd" pointers may be HOST or DEVICE addresses (detected with cudaPointerGetAttributes); host buffers
 *     are staged through the context's stream.  Output buffers are caller-owned.
 *   - all work is enqueued on the context's stream (mpb_ctx_set_stream; default: the legacy stream); calls
 *     that fill HOST outputs synchronise that stream before returning, calls that fill DEVICE outputs do not.
 *   - alignment cells are 4-bit base sets: A=1, C=2, G=4, T=8, IUPAC code = OR of its bases, gap = 0
 *     (core:441-455 parse_seq maps every other character, N included, to '-').
 *   - primer length k: 3 <= k <= 27 (haplotype keys are 64-bit; see DESIGN.md "keys").
 */
#ifndef MPB200_H
#define MPB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPB_ABI_VERSION 3
#define MPB_MAX_K 27
#define MPB_MAX_EXPANSIONS 65536 /* expansions of one k-mer window of one sequence */

#define MPB_OK 0
#define MPB_EINVAL (-1)    /* bad argument */
#define MPB_ECUDA (-2)     /* CUDA runtime error (message has the cudaError string) */
#define MPB_ENOMEM (-3)    /* device allocation failed */
#define MPB_EOVERFLOW (-4) /* haplotype table full: retry mpb_hist_build with a larger log2_cap */
#define MPB_EEXPAND (-5)   /* a window holds more than MPB_MAX_EXPANSIONS expansions / a row has < k bases */

typedef struct mpb_ctx mpb_ctx;   /* one CUDA device + stream */
typedef struct mpb_msa mpb_msa;   /* an alignment resident in HBM as base bit-planes */
typedef struct mpb_hist mpb_hist; /* per-window haplotype tables of one window batch */

int mpb_abi_version(void);
const char* mpb_last_error(void);
int mpb_device_count(void);

int mpb_ctx_create(int device, mpb_ctx** out);
void mpb_ctx_destroy(mpb_ctx* ctx);
int mpb_ctx_set_stream(mpb_ctx* ctx, void* cuda_stream);
int mpb_ctx_sync(mpb_ctx* ctx);
/* number of kernels this context has launched so far (bench.py's "gpu_launches") */
int64_t mpb_ctx_launches(mpb_ctx* ctx);
/* stream-ordered device memory owned by the caller (results that stay in HBM between calls) */
int mpb_dev_alloc(mpb_ctx* ctx, int64_t bytes, void** out);
void mpb_dev_free(mpb_ctx* ctx, void* p);
/* copy between host / device memory on the context's stream; returns after the copy has completed */
int mpb_ctx_memcpy(mpb_ctx* ctx, void* dst, const void* src, int64_t bytes);
/* set `bytes` bytes of device memory to `value` on the context's stream; returns after it has completed */
int mpb_ctx_memset(mpb_ctx* ctx, void* dst, int value, int64_t bytes);

/* Profiling: when enabled every kernel launch is bracketed by CUDA events on the context's stream.
 * mpb_ctx_profile_read sums duration (ms), launch count and algorithmic work units (candidate x sequence
 * evaluations for "k_scan", extracted k-mers for "k_hist") of the launches of one kernel since the last clear;
 * kernel == NULL clears the records. */
int mpb_ctx_profile(mpb_ctx* ctx, int enable);
int mpb_ctx_profile_read(mpb_ctx* ctx, const char* kernel, double* ms, int64_t* launches, double* units);

/* ---- alignment ---------------------------------------------------------------------------------------
 * core:441-455 parse_seq keeps the alignment as {id: string}; here it lives in HBM as four bit-planes
 * (A,C,G,T) per 32-column word, sequence index fastest: planes[col_word][plane][seq].
 * packed4_hd: n_seq rows of row_bytes bytes, two cells per byte, low nibble = even column.
 * lens (host, may be NULL = all n_col): row lengths of a ragged (unaligned) input such as test_data/test.fa.
 */
int mpb_msa_upload(mpb_ctx* ctx, const uint8_t* packed4_hd, int64_t n_seq, int64_t n_col, int64_t row_bytes,
                   const int32_t* lens, mpb_msa** out);
void mpb_msa_free(mpb_msa* msa);
int64_t mpb_msa_nseq(const mpb_msa* msa);

/* Sequence-sharded runs: global index of this shard's first sequence (enters the first-seen order of the tables). */
int mpb_msa_set_row0(mpb_msa* msa, int64_t row0);

/* core:617-627 seq_attribute, per-sequence part: number of leading gap cells and length after stripping
 * trailing gaps.  The two quantiles (core:629-633) are taken by the host. */
int mpb_seq_attr(mpb_msa* msa, int32_t* lead_gaps_hd, int32_t* rstrip_len_hd);

/* Entropy prefilter.  For every window: s0 = number of items the reference's total entropy runs over (expansions of
 * cover rows + gap rows), s1 = sum(c log2 c) over a 65536-bin coarsening of their k-mers (a 16-bit hash of the 2-bit
 * bases of all cells).  (s0 log2 N - s1) / N is a LOWER bound of "Entropy of total" (core:602-614) because merging categories
 * cannot raise sum(-p log p); a window whose bound exceeds the gate can be dropped without building its table. */
int mpb_window_prefilter(mpb_msa* msa, int k, int v, const int32_t* win_pos, int32_t nw, double* s0_hd, double* s1_hd);

/* The same two attributes as histograms over the values 0..n_col (hd arrays of n_col+1 int64): an order statistic
 * needs no sort, and sequence shards add their histograms. */
int mpb_seq_attr_hist(mpb_msa* msa, int64_t* lead_hist_hd, int64_t* rstrip_hist_hd);

/* ---- window haplotype tables: core:651-711 (sequence loop of get_primers) ---------------------------------
 * For every window start win_pos[i] (host array) extract each sequence's k-mer with the reference's
 * terminal-gap patching, expand IUPAC cells, and count haplotypes into an open-addressing table per window
 * (cover / gap_sequence dictionaries of the reference).  log2_cap = 0 picks 2^ceil(log2(2*n_seq+64)).
 * Any start 0 <= win_pos[i] < n_col is accepted.  A window with win_pos[i] + k > n_col (or past a ragged row's end)
 * takes the reference's left extension (core:683-687): the row's cells from win_pos[i] on, patched, preceded by the
 * bases left of them; a row without enough bases there fails the call with MPB_EEXPAND.
 */
int mpb_hist_build(mpb_msa* msa, int k, int v, const int32_t* win_pos, int32_t nw, int log2_cap, mpb_hist** out);
void mpb_hist_free(mpb_hist* h);

/* The same tables, empty: the OWNER tables of a sequence-sharded run (SURVEY.md 8e) hold the windows one rank owns and
 * are filled with the entries of every shard through mpb_hist_merge; gap-row counters come in through
 * mpb_hist_add_counts (host arrays of nw, already summed over the shards). */
int mpb_hist_create_empty(mpb_msa* msa, int k, int v, const int32_t* win_pos, int32_t nw, int log2_cap, mpb_hist** out);
int mpb_hist_add_counts(mpb_hist* h, const int64_t* gap_n, const int64_t* n_iupac_gap);

/* Counters kept while building (host arrays of nw, any may be NULL): gap rows, gap rows holding IUPAC cells, distinct
 * table entries — what a sequence shard needs to size mpb_hist_export without a pass over its tables. */
int mpb_hist_counts(mpb_hist* h, int64_t* gap_n, int64_t* n_iupac_gap, int64_t* n_entries);

/* Copy all entries of the windows with sel[i] != 0 (host array) into compact arrays: window i's entries land in
 * [win_off[i], win_off[i+1]) (host array of nw+1, sized by the caller from mpb_hist_stats' nuniq; unordered). */
int mpb_hist_export(mpb_hist* h, const uint8_t* sel, const int64_t* win_off, uint64_t* keys_hd, uint32_t* cnt_hd,
                    uint64_t* first_hd);

/* The same with explicit placement: the entries of window sel_idx[i] (host array, any order) land in
 * [start[i], start[i] + room[i]) of the hd arrays (total elements).  A sequence shard lays its windows out by owning
 * rank so that one all-to-all moves them.  Does not synchronise when the outputs are device memory. */
int mpb_hist_export_at(mpb_hist* h, int32_t n_sel, const int32_t* sel_idx, const int64_t* start, const int64_t* room,
                       int64_t total, uint64_t* keys_hd, uint32_t* cnt_hd, uint64_t* first_hd);

/* Insert foreign (key, count, first) triples into the tables (multi-GPU merge of per-rank tables).
 * win_off (host, nw+1) delimits the triples of each window inside the hd arrays. */
int mpb_hist_merge(mpb_hist* h, const int64_t* win_off, const uint64_t* keys_hd, const uint32_t* cnt_hd,
                   const uint64_t* first_hd);

/* One pass over the occupied slots of every window: mpb_hist_stats and mpb_hist_tensors together (HOST outputs, any
 * may be NULL; freq / nn for ALL windows of the batch).  The tensors also stay on the device for mpb_walk_dev_begin. */
int mpb_hist_summary(mpb_hist* h, int64_t* gap_n, double* ent, int64_t* nuniq, uint64_t* mm_key, int64_t* mm_cnt,
                     uint64_t* mm_first, int64_t* n_iupac_gap, int64_t* freq, int64_t* nn);

/* The same with n_seg = m * nw segments (seg_off[n_seg + 1], host): segment s belongs to window s % nw — what an owner
 * receives from m source ranks in one all-to-all. */
int mpb_hist_merge_segments(mpb_hist* h, int32_t n_seg, const int64_t* seg_off, const uint64_t* keys_hd,
                            const uint32_t* cnt_hd, const uint64_t* first_hd);

/* Per-window summary (HOST outputs, any may be NULL):
 *   gap_n[nw]        sequences with more than v gaps (gap_sequence_number, core:689-691)
 *   ent[nw*4]        sum(c), sum(c*log2 c) over cover haplotypes; the same two sums over gap k-mers
 *                    (ingredients of core:602-614 entropy; the host rounds / re-derives exactly)
 *   nuniq[nw*3]      distinct cover haplotypes, distinct gap k-mers, distinct gap-free cover haplotypes
 *   mm_key/mm_cnt/mm_first[nw]  most frequent gap-free haplotype, first seen wins ties (core:595-600)
 *   n_iupac_gap[nw]  gap rows holding IUPAC cells (not in the table; listed by mpb_hist_exceptions)
 */
int mpb_hist_stats(mpb_hist* h, int64_t* gap_n, double* ent, int64_t* nuniq, uint64_t* mm_key, int64_t* mm_cnt,
                   uint64_t* mm_first, int64_t* n_iupac_gap);

/* core:541-554 state_matrix and core:556-577 trans_matrix for the windows with sel[i] != 0 (host array):
 *   freq[nw*4*k]       freq[w][b][col]  expansion rows with base b (A,C,G,T) at column col
 *   nn[nw*(k-1)*16]    nn[w][col][x*4+y] expansion rows with x at col and y at col+1
 */
int mpb_hist_tensors(mpb_hist* h, const uint8_t* sel, int64_t* freq_hd, int64_t* nn_hd);

/* All entries of window w, unordered: keys (see DESIGN.md for the encoding), counts, first-seen order
 * (seq_index << 16 | expansion_index).  *n_out receives the number of entries (<= max_n). */
int mpb_hist_dump(mpb_hist* h, int32_t w, int64_t max_n, uint64_t* keys_hd, uint32_t* cnt_hd, uint64_t* first_hd,
                  int64_t* n_out);

/* Number of DISTINCT gap-free haplotypes of window q_win[i] (index into the batch) that are expansions of the
 * degenerate pattern q_allow[i*4 + b] (bit col set = base b allowed at col).  Used for nonsense_primer_number
 * (core:846). */
int mpb_hist_match(mpb_hist* h, const int32_t* q_win, const uint32_t* q_allow, int32_t nq, int64_t* distinct_hd);

/* (window index, sequence index) pairs of gap rows that hold IUPAC cells, at most max_n pairs */
int mpb_hist_exceptions(mpb_hist* h, int64_t max_n, int32_t* win_idx, int32_t* seq_idx, int64_t* n_out);

/* ---- the candidate scan: core:1103-1130 mis_primer_check + core:229-233 Y_distance ---------------------------
 * One evaluation = one candidate primer against one sequence's (patched, expanded) k-mer of the candidate's
 * window.  cand_pos[nc] window start columns (ascending), cand_allow[nc*4] allowed-base bit masks.
 * fmask / rmask: bit i set = a mismatch at primer position i disqualifies F / R coverage (core:1091-1101).
 *   counts[nc*3]   expansion rows with 0 mismatches | 1..v mismatches and none at an F-strict position |
 *                  the same for R      (perfect coverage, F_mis_cover, R_mis_cover of the reference)
 *   bits_slot[nc]  (host, may be NULL) >= 0: also write per-sequence bit vectors for this candidate into
 *                  bits[slot*3*words .. ): F non-cover, R non-cover, gap row; words = ceil(n_seq/32)
 */
int mpb_scan(mpb_msa* msa, int k, int v, uint32_t fmask, uint32_t rmask, const int32_t* cand_pos_hd,
             const uint32_t* cand_allow_hd, int64_t nc, int64_t* counts_hd, const int32_t* bits_slot,
             uint32_t* bits_hd);

/* The same evaluation on the COLUMN view of the alignment (one thread = one candidate against 32 sequences: the
 * mismatch word of a position is the complement of the OR of the allowed bases' column-plane words, mismatches are
 * counted by a carry-save adder on the 32 lanes, the 3'-end rules are ORs over the strict positions).  Rows whose
 * window is not the plain column cut (terminal-gap patching, IUPAC cells, ragged end: recorded per window by
 * mpb_hist_build) are evaluated from their stored patched windows.  Candidates name a window of h's batch.
 *   cands[nc]      hd; trial >= 0 also counts the perfect matches that carry base (trial >> 8) at position
 *                  (trial & 255): the reference's coverage_renew look-up (core:954-956) folded into its parent
 *   counts[nc*4]   hd: perfect | F_mis | R_mis | trial perfect  (mpb_scan's first three)
 *   bits_slot / bits   as mpb_scan (bits hd, slots host)
 * variation (h's v) must be <= 15. */
typedef struct mpb_cand {
    int32_t win;   /* index into the window batch of the mpb_hist */
    int32_t trial; /* position | base << 8, or -1 */
    uint32_t allow[4];
} mpb_cand;
int mpb_cscan(mpb_hist* h, uint32_t fmask, uint32_t rmask, const mpb_cand* cands_hd, int64_t nc, int64_t* counts_hd,
              const int32_t* bits_slot, uint32_t* bits_hd);

/* Exhaustive exact search (extract_PCR_product_V1.py:189-216 get_PCR_PRODUCT; SURVEY.md 8f-4): every position of every
 * sequence of the alignment handle (an unaligned FASTA uploaded as ragged rows) against n_pat degenerate patterns
 * (allow[n_pat*4] allowed-base masks, lens[n_pat] <= 32; host arrays).  Host outputs of capacity max_hits receive
 * (pattern, sequence, position) of every occurrence of an expansion, unordered; *n_hits may exceed max_hits (then call
 * again with more room).  A cell that is not exactly one base (IUPAC code, N, gap) never matches, as in the reference's
 * plain-text search. */
int mpb_pattern_hits(mpb_msa* msa, int32_t n_pat, const uint32_t* allow, const int32_t* lens, int64_t max_hits,
                     int32_t* hit_pat, int32_t* hit_row, int32_t* hit_pos, int64_t* n_hits);

/* The same search with up to v mismatches per site (primer_coverage.py, the mismatch rule of mis_primer_check
 * core:1103-1130): a site of pattern p at position x of a row is reported when the pattern lies inside the row's lens,
 * at most v of its cells mismatch (a cell that is not exactly one allowed base mismatches) and none of the mismatches
 * falls on a position whose bit is set in strict[p] (host array).  hit_mis receives the site's mismatch count; the other
 * outputs and the capacity rule are those of mpb_pattern_hits.  0 <= v <= 15 and v < lens[p] for every pattern. */
int mpb_pattern_sites(mpb_msa* msa, int32_t n_pat, const uint32_t* allow, const int32_t* lens, const uint32_t* strict,
                      int32_t v, int64_t max_hits, int32_t* hit_pat, int32_t* hit_row, int32_t* hit_pos, int32_t* hit_mis,
                      int64_t* n_hits);

/* In-silico PCR over every primer combination (primer_specificity.py).  The handle's rows are overlapping cuts of one
 * stream: row r holds stream columns [r*stride, r*stride + n_col).  The patterns (allow / lens / strict / v as in
 * mpb_pattern_sites) belong to primers: pattern p is a LEFT site of primer pat_primer[p] (pat_side[p] == 0: the primer
 * binds on the stored strand) or a RIGHT site (1: its reverse complement binds).  A site is kept when it starts in the
 * first `stride` columns of its row and lies inside one of the n_rec records (stream offsets rec_off[] ascending and
 * lengths rec_len[], relative to row 0 of the handle).  A product (i, j) is a left site of i at x and a right site of j
 * at y in one record with y >= x + L_i and y + L_j - x in [lo, hi]; a group is (record, i, j) with at least one
 * product, and its best product has the fewest total mismatches, then the smallest length, then the smallest x.
 * Sites, products and groups stay on the device; memory is bounded by sites + groups (left sites are joined in chunks
 * of at most `chunk`, 0 = default).  Host outputs:
 *   comb[(i*n_primer + j)*3 + {0,1,2}]  products, groups (targets), groups whose best product has no mismatch;
 *   uni[2]   records with a group of a combination whose list[i*n_primer + j] is set, and those with a perfect one;
 *   rows[max_rows*8]  the first max_rows listed groups in (record, i, j) order: record, i, j, start, length, left
 *            mismatches, right mismatches, products (start 0-based on the record); *n_listed = all listed groups;
 *   stats[4] search hits, left sites, right sites, groups.
 * Limits (MPB_EINVAL): 1 <= n_primer <= 1024, 0 < lo <= hi <= 2^23 - 1, records shorter than 2^32, a stream shorter
 * than 2^43 columns. */
int mpb_pattern_products(mpb_msa* msa, int32_t n_pat, const uint32_t* allow, const int32_t* lens, const uint32_t* strict,
                         int32_t v, const int32_t* pat_primer, const int32_t* pat_side, int32_t n_primer, int64_t stride,
                         int32_t n_rec, const int64_t* rec_off, const int64_t* rec_len, int32_t lo, int32_t hi,
                         const uint8_t* list, int64_t chunk, int64_t max_rows, int64_t* comb, int64_t* uni, int64_t* rows,
                         int64_t* n_listed, int64_t* stats);

/* Coverage of every pair by its own two patterns (primer_select.py).  Rows, stride, records and allow / lens / strict / v
 * as in mpb_pattern_products; the n_pat = 4 * pairs patterns are in primer_coverage's Panel order: F, RC(R), R, RC(F)
 * of pair 0, then of pair 1, ...  An amplicon of pair q is a site of pattern 4q at x and of 4q+1 at y (+ strand), or of
 * 4q+2 at x and 4q+3 at y (- strand), in one record, with y >= x + L(left) and y + L(right) - x in [lo, hi].  The call
 * ORs bit r of amp[q*words + r/32] for every record r where pair q has an amplicon, and the same bit of perf[...] when one
 * of them has no mismatch on either site (amp / perf: device memory the caller zeroes; offset them for a block of
 * pairs).  max_sites: the search's first capacity (0: 2^24); when the search finds more sites it runs once more with
 * room for all of them, so a caller that knows the count (from the previous call of a block loop) saves that second
 * pass.  stats[3]: search hits, left sites, right sites.  Device memory is bounded by the sites of the call; products
 * are never stored.  Limits (MPB_EINVAL): n_pat a positive multiple of 4, n_rec < 2^31, words >= ceil(n_rec / 32),
 * 0 < lo <= hi, 0 <= max_sites <= 2^31, every record ending inside the rows (rec_off + rec_len <= rows * stride),
 * bits(n_pat) + bits(rows * stride) + 4 <= 64 (the site key). */
int mpb_pattern_cover(mpb_msa* msa, int32_t n_pat, const uint32_t* allow, const int32_t* lens, const uint32_t* strict,
                      int32_t v, int64_t stride, int32_t n_rec, const int64_t* rec_off, const int64_t* rec_len, int32_t lo,
                      int32_t hi, int64_t words, uint32_t* amp, uint32_t* perf, int64_t max_sites, int64_t* stats);
/* The greedy step over a coverage matrix amp / perf [n_rows][words] (device, words a positive multiple of 4, 16-byte
 * aligned) and the covered vectors covered / covered_perfect [words] (device): for the rows cand[n_cand] (host),
 * gains[2i] = popcount(amp[cand[i]] & ~covered) and gains[2i+1] = popcount(perf[cand[i]] & ~covered_perfect) (host or
 * device).  Rows that are not listed are not read. */
int mpb_cover_gains(mpb_ctx* ctx, const uint32_t* amp, const uint32_t* perf, int64_t n_rows, int64_t words,
                    const uint32_t* covered, const uint32_t* covered_perfect, const int32_t* cand, int64_t n_cand,
                    int64_t* gains);
/* covered |= amp[row], covered_perfect |= perf[row] (the arrays of mpb_cover_gains) */
int mpb_cover_take(mpb_ctx* ctx, const uint32_t* amp, const uint32_t* perf, int64_t n_rows, int64_t words, int64_t row,
                   uint32_t* covered, uint32_t* covered_perfect);

/* A resident site list: the filtered sites of every pattern of a panel (n_pat = 4 * pairs, Panel order, lens[n_pat]
 * host) over one set of records (rec_off / rec_len [n_rec] host, as in mpb_pattern_cover) in a stream of n_pos columns,
 * kept in device memory for the joins of primer_select.py --cross / --background.  One 64-bit key per site:
 * stream position << (bits(n_pat) + 4) | pattern << 4 | mismatches.  Limits (MPB_EINVAL): bits(n_pat) + bits(n_pos) + 4
 * <= 64, every record ending inside n_pos. */
typedef struct mpb_site_list mpb_site_list;
int mpb_site_list_create(mpb_ctx* ctx, int32_t n_pat, const int32_t* lens, int64_t n_pos, int32_t n_rec,
                         const int64_t* rec_off, const int64_t* rec_len, mpb_site_list** out);
void mpb_site_list_destroy(mpb_site_list* list);
/* mpb_pattern_cover on the patterns pat0 .. pat0 + n_pat - 1 of the list (pat0 a multiple of 4; lens and records equal
 * to the list's), with its filtered sites also appended to the list: the same single search.  amp = perf = NULL only
 * searches and keeps (no sort, no join; words is not read).  A list that cannot grow fails with MPB_ENOMEM and a message
 * that names the bytes. */
int mpb_pattern_cover_keep(mpb_msa* msa, int32_t n_pat, const uint32_t* allow, const int32_t* lens, const uint32_t* strict,
                           int32_t v, int64_t stride, int32_t n_rec, const int64_t* rec_off, const int64_t* rec_len,
                           int32_t lo, int32_t hi, int64_t words, uint32_t* amp, uint32_t* perf, int64_t max_sites,
                           int64_t* stats, mpb_site_list* list, int32_t pat0);
/* Sort every kept key once (stream order; a sealed list takes no more sites): *n_sites = the list's sites. */
int mpb_site_list_seal(mpb_site_list* list, int64_t* n_sites);
/* The first min(cap, sites) keys in list order into keys[] (host); *n_sites = the list's sites. */
int mpb_site_list_keys(mpb_site_list* list, int64_t cap, uint64_t* keys, int64_t* n_sites);
/* The products between the taken pair `pair` (t) and every pair c whose bit c of eligible[ceil(pairs / 32)] (host) is set,
 * on a sealed list: a left site of primer i at x and a right site of primer j at y in one record, with y >= x + L_i and
 * y + L_j - x in [lo, hi], i of one pair and j of the other.  bits[pairs] (host): bit side << 2 | primer of c << 1 |
 * primer of t of byte c (side 0: t's primer is the left one; primer 0 = F, 1 = R). */
int mpb_sites_cross(mpb_site_list* list, int32_t lo, int32_t hi, int32_t pair, const uint32_t* eligible, uint8_t* bits);
/* Each pair's products of its own primers on a sealed list: bits[pairs] (host), bit left primer << 1 | right primer of
 * byte q set when pair q's (F, F), (F, R), (R, F) or (R, R) has a product. */
int mpb_sites_own(mpb_site_list* list, int32_t lo, int32_t hi, uint8_t* bits);

/* Per (window, sequence) haplotype key, for the JSON side files (core:1172-1176): the table key of the
 * sequence's k-mer, MPB_KEY_IUPAC for rows whose window holds IUPAC cells. out[nw*n_seq]. */
#define MPB_KEY_IUPAC 0xFFFFFFFFFFFFFFFEull
#define MPB_KEY_EMPTY 0xFFFFFFFFFFFFFFFFull
#define MPB_KEY_BASE5 (1ull << 54) /* keys >= this are base-5 numbers of k-mers that hold gaps */
int mpb_seqkeys(mpb_msa* msa, int k, const int32_t* win_pos, int32_t nw, uint64_t* out_hd);

/* ---- nearest-neighbour Tm: core:249-261 Calc_deltaH_deltaS + core:328-335 ---------------------------------
 * seqs2bit[n*k] bases 0..3 (A,C,G,T).  consts = {R*ln(C/4e9), R*ln(C/1e9), salt correction} evaluated by the
 * host with the reference's expressions; tm_out[n] unrounded fp64 (the host applies Python round()).
 */
int mpb_tm(mpb_ctx* ctx, const uint8_t* seqs2bit_hd, int k, int64_t n, const double* consts3, double* tm_hd,
           double* dh_hd, double* ds_hd);

/* The same for degenerate primers given as base sets (sets[n*32], one byte per position, hd): sums[n] = sum over the
 * expansions of round(Tm, 2) in hundredths of a degree (exact integers), ties[n] = expansions left out because their Tm
 * sits within 1e-6 of a rounding tie (the caller replays such a primer with Python's round()).  Host outputs. */
int mpb_tm_sets(mpb_ctx* ctx, const uint8_t* sets_hd, int k, int32_t n, const double* consts3, int64_t* sums, int32_t* ties);

/* ---- per-window control logic: seeds core:579-600, NN-array refinement walk core:860-1089, NM-vs-MM core:816 ----------
 * The logic lives once in csrc/mpb_walk_core.h and compiles for host and device.
 *
 * mpb_walk_dev_*: the product path.  Tracks (two per window: Viterbi seed and, when different, the most frequent
 * haplotype) are resident in HBM; every round is a chain of kernels on the context's stream — advance all tracks with
 * the previous round's counts and emit the next candidates, plan them, column scan, special rows — with NO host
 * round trip: the host only enqueues.  In sequence-sharded runs the caller all-reduces the count vector between
 * mpb_walk_dev_scan and the next mpb_walk_dev_advance (counts_dev is caller-visible device memory).
 *   n_win, win_idx[n_win]      the windows that walk (indices into h's batch), host array
 *   cover_number[n_win], mm_key[n_win]   host arrays (MPB_KEY_EMPTY: no gap-free haplotype)
 *   freq_hd[n_win*4*k], nn_hd[n_win*(k-1)*16]  hd, or NULL = h's own summary tensors (mpb_hist_summary) at win_idx
 * mpb_walk_dev_round = advance + scan.  Rounds after the last live track are no-ops.
 * mpb_walk_dev_finish synchronises and returns mpb_walk's outputs. */
typedef struct mpb_walk_dev mpb_walk_dev;
int mpb_walk_dev_begin(mpb_hist* h, int dnum, int degeneracy, uint32_t fmask, uint32_t rmask, int32_t n_win,
                       const int32_t* win_idx, const int64_t* cover_number, const uint64_t* mm_key, const int64_t* freq_hd,
                       const int64_t* nn_hd, mpb_walk_dev** out);
int mpb_walk_dev_advance(mpb_walk_dev* w);
int mpb_walk_dev_scan(mpb_walk_dev* w);
int mpb_walk_dev_round(mpb_walk_dev* w);
/* device address and capacity (int64 elements) of the count vector of the current round, for the caller's all-reduce */
int mpb_walk_dev_counts(mpb_walk_dev* w, void** counts_dev, int64_t* n_elems);
/* number of live tracks after the last advance that has completed (-1: none yet); never blocks */
int64_t mpb_walk_dev_live(mpb_walk_dev* w);
int mpb_walk_dev_max_rounds(mpb_walk_dev* w);
/* block until the live-track count after advance number `round` (0-based) is known */
int mpb_walk_dev_wait(mpb_walk_dev* w, int round, int64_t* live);
/* single-process driver: advance / scan until no track is live, the host at most `lag` rounds ahead of the device */
int mpb_walk_dev_run(mpb_walk_dev* w, int lag, int64_t* rounds);
int mpb_walk_dev_finish(mpb_walk_dev* w, uint8_t* out_sets, int64_t* out_counts, uint8_t* out_seeds, int64_t* out_seed_cover,
                        int32_t* out_ntracks, int64_t trace_cap, uint8_t* trace_sets, int64_t* trace_off, int64_t* stats);
void mpb_walk_dev_free(mpb_walk_dev* w);

/* ---- peer-memory all-reduce for sequence-sharded walks (no counterpart in the reference; SURVEY.md 8e) --------------
 * One process (or thread) per GPU.  Every rank creates a group member, publishes its 128-byte handle, collects the
 * handles of all ranks in rank order (through whatever channel the host has: torch.distributed, MPI, a file) and
 * connects.  The receive buffers are opened through CUDA IPC over NVLink (same-process members are used by address).
 * mpb_walk_dev_set_peer makes mpb_walk_dev_run sum the count vector over the ranks after every scan with ONE
 * single-block kernel on the walk's stream (push to every peer, signal, wait, sum) instead of a collective-library call
 * from the host per round.  cap_elems = capacity of the vector in int64 elements (4 per candidate of a round). */
#define MPB_PEER_MAX_WORLD 8
#define MPB_PEER_HANDLE_BYTES 128
typedef struct mpb_peer mpb_peer;
int mpb_peer_create(mpb_ctx* ctx, int rank, int world, int64_t cap_elems, mpb_peer** out);
int mpb_peer_handle(mpb_peer* p, void* handle_out /* MPB_PEER_HANDLE_BYTES */);
int mpb_peer_connect(mpb_peer* p, const void* handles /* world x MPB_PEER_HANDLE_BYTES, rank order */);
int64_t mpb_peer_cap(mpb_peer* p);
/* in-place sum over the ranks of data_dev[0..n) (device memory); collective: same calls in the same order on all ranks */
int mpb_peer_allreduce(mpb_peer* p, int64_t* data_dev, int64_t n);
/* the two halves of a round as separate calls — phases 1: push + signal, 2: wait + sum, 3: both — so that one stream can
 * play every rank of a group in turn (all ranks' phase 1, then all ranks' phase 2) */
int mpb_peer_allreduce_phases(mpb_peer* p, int64_t* data_dev, int64_t n, int phases);
void mpb_peer_free(mpb_peer* p);
/* the walk's rounds all-reduce their counts through `peer` (NULL: back to the caller's own all-reduce between
 * mpb_walk_dev_scan and mpb_walk_dev_advance); fails when a round's vector could exceed the group's capacity */
int mpb_walk_dev_set_peer(mpb_walk_dev* w, mpb_peer* peer);

/* mpb_walk: the same walk driven from the host with the scan as a callback (no device code, no CUDA calls): the CPU
 * tests run it against a stand-in scan.  Candidates name windows 0..n_win-1.
 *   out_sets[n_win*32]       final primer (4-bit sets) of the chosen track
 *   out_counts[n_win*5]      optimal_coverage_init, F_mis_cover_cover, R_mis_cover_cover (core:917-918 before the
 *                            sum), chosen track (0 = first / NM, 1 = MM), perfect_coverage of the final primer (core:853)
 *   out_seeds[n_win*2*32]    seed bases (0..3) of the tracks; out_seed_cover[n_win*2] cover[seed] (-1: no such track)
 *   out_ntracks[n_win]       1 or 2
 *   trace_sets[trace_cap*32], trace_off[n_win+1]   every primer handed to mis_primer_check, in call order
 *   stats[3]                 scan rounds, candidates scanned, trace length
 */
typedef int (*mpb_scan_cb)(void* user, const mpb_cand* cands, int64_t nc, int64_t* counts /* nc*4 */);
int mpb_walk(int k, int v, int dnum, int degeneracy, int32_t n_win, const int64_t* cover_number, const int64_t* freq,
             const int64_t* nn, const uint64_t* mm_key, mpb_scan_cb scan, void* user, uint8_t* out_sets,
             int64_t* out_counts, uint8_t* out_seeds, int64_t* out_seed_cover, int32_t* out_ntracks, int64_t trace_cap,
             uint8_t* trace_sets, int64_t* trace_off, int64_t* stats);

/* Tm (mean over expansions of the rounded per-expansion Tm, core:849-852; k_tm on the device), GC content and the
 * di-nucleotide / hairpin filters (core:387-416, 507-521) of n primers sets[n*32] of length k (host arrays).
 * flags: 1 GC outside [gc_lo, gc_hi], 2 di-nucleotide repeat, 4 hairpin, 64 / 128: the Tm / GC mean sits on a
 * rounding tie that double arithmetic cannot decide — the caller replays that value exactly. */
int mpb_primer_props(mpb_ctx* ctx, const uint8_t* sets, int k, int32_t n, double gc_lo, double gc_hi, int distance,
                     const double* tm_consts3, double* tm_avg, double* gc, int32_t* flags, int32_t* deg, int32_t* ndeg);

/* The reference's raw k-mer of (sequence, window) pairs — window cut, terminal-gap patching and the left extension of
 * a short row, core:666-687 — read from the HOST copy of the alignment (nibble-packed rows as mpb_msa_upload takes them:
 * cell c of a row = (row[c / 2] >> 4 * (c & 1)) & 15; lens NULL = every row n_col cells).  Pure host code, no context:
 * used for the handful of gap rows holding IUPAC cells, which the device tables do not store (mpb_hist_exceptions).
 * cells[n*32]: 4-bit base sets of the k-mer, zero padded; out_len[n]: its length (< k when the row cannot supply k
 * cells). */
int mpb_window_cells(const uint8_t* packed, int64_t row_stride, const int32_t* lens, int32_t n_col, int k, int64_t n,
                     const int64_t* seq, const int32_t* pos, uint8_t* cells, int32_t* out_len);

/* ---- pair coverage: get_multiPrime.py:560-569 ---------------------------------------------------------------------
 * uf / ur [n_rows*words]: per-candidate bit vectors of the sequences the forward / reverse use of that candidate leaves
 * uncovered (gap rows included), in mpb_scan's bit layout.  uncovered[q] = popcount(uf[pf[q]] | ur[pr[q]]). */
int mpb_pair_cover(mpb_ctx* ctx, const uint32_t* uf_hd, const uint32_t* ur_hd, int32_t n_rows, int32_t words,
                   const int32_t* pf_hd, const int32_t* pr_hd, int64_t n_pairs, int32_t* uncovered_hd);

/* The same straight from the scan's bit vectors bits[n_rows*3*words] (hd; mpb_cscan layout: F non-cover, R non-cover,
 * gap rows per candidate): uncovered[q] = popcount(F[pf] | gap[pf] | R[pr] | gap[pr]).  SURVEY.md 8f-1: the pairing
 * step reads the scan's output where it lies, no JSON side files in between. */
int mpb_pair_cover3(mpb_ctx* ctx, const uint32_t* bits_hd, int32_t n_rows, int64_t words, const int32_t* pf_hd,
                    const int32_t* pr_hd, int64_t n_pairs, int32_t* uncovered_hd);

/* ---- primer-dimer predicates: core:457-503 dimer_check, finDimer_V4.py:191-224 ---------------------------------
 * sets[n*32] 4-bit base sets of n primers (one byte per position, row stride 32), lens[n] (host arrays).
 * Ends = suffixes of length min(max_end, len) .. min_end (max_end <= 0: len + max_end .. min_end, the
 * get_Maxprimerset_V1.3.py:149-154 variant), longest first, each expanded in product order
 * (core:457-464 current_end after the stable length sort of core:489).
 * loss_table[33*33*33] (host): loss_table[(len*33+gc)*33+d2] != 0 when the reference's Loss test passes for an end of
 * that length / GC count at distance d2 (the host evaluates core:192-193 itself, so >= vs > and the threshold are its
 * business).  dg_consts[24] (host): stacking terms of core:466-485, see mpb_dimer.cu.  init_both = 0 selects the
 * get_multiPrime.py:400-416 variant of dG (initiation term of the first base only).
 */
typedef struct mpb_dimer mpb_dimer;
int mpb_dimer_prepare(mpb_ctx* ctx, const uint8_t* sets, const int32_t* lens, int32_t n, int min_end, int max_end,
                      int init_both, const uint8_t* loss_table, const double* dg_consts, mpb_dimer** out);
void mpb_dimer_free(mpb_dimer* d);
/* expansion / end offsets per primer (host arrays of n+1) */
int mpb_dimer_counts(mpb_dimer* d, int64_t* off_p, int64_t* off_e);
/* For each pair (pi[q], pj[q]) (host arrays): first_hit[q] = e_index * n_expansions(pj) + p_index of the first
 * (end of pi, expansion of pj) in reference order that forms a dimer, or -1; hit_d2[q] its distance 2. */
int mpb_dimer_pairs(mpb_dimer* d, const int32_t* pi, const int32_t* pj, int64_t n_pairs, int64_t* first_hit,
                    int32_t* hit_d2);

/* All pairs (i, j >= i) with i in [row0, row1): finDimer_V4.py:191-224.  Host output arrays of capacity max_hits
 * receive the pairs that form a dimer (sorted by i, j), the first-hit order index and its distance 2; *n_tested the
 * pairs that survived the 5-mer prefilter.  Needs min_end == 5 at mpb_dimer_prepare. */
int mpb_dimer_grid(mpb_dimer* d, int32_t row0, int32_t row1, int64_t max_hits, int32_t* hit_i, int32_t* hit_j,
                   int64_t* hit_order, int32_t* hit_d2, int64_t* n_hits, int64_t* n_tested);

/* ---- pool assignment: multiprime_b200/primer_pools.py states the search rule -------------------------------------
 * w[n*n] (host): symmetric conflict weights of n pairs with a zero diagonal.  Restarts r in [r0, r1) of the tabu search
 * into n_pools balanced pools, each independent of the others: best_cost[r - r0] is the lowest cost the restart
 * reached, best_step[r - r0] the first step at which it did, assign[(r - r0)*n + a] the pool of pair a at that step
 * (host arrays).  Limits (MPB_EINVAL): 1 <= n <= 512, 1 <= n_pools <= 32, n_pools <= n, 0 <= r0 <= r1 <= 2^24,
 * 0 <= iterations <= 2^20 - 1, w symmetric with a zero diagonal. */
int mpb_pool_search(mpb_ctx* ctx, int32_t n, int32_t n_pools, const uint8_t* w, uint64_t seed, int64_t r0, int64_t r1,
                    int32_t iterations, int64_t* best_cost, int32_t* best_step, uint8_t* assign);

#ifdef __cplusplus
}
#endif
#endif /* MPB200_H */
