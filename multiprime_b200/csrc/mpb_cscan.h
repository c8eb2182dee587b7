// mpb_cscan.h — internal interface of the column scan (mpb_cscan.cu), shared with the device walk (mpb_walk_dev.cu)
#pragma once
#include <stdint.h>

#include "mpb200.h"
#include "mpb_host.h"

#define CSCAN_PLAN_WORDS 384        // header 8 + 9 triples x 4 + 108 degenerate entries + 2 x 108 strict entries, rounded
#define CSCAN_NONE 0xFFFFFFFFu
#define MPB_ERR_BAD_CAND 8

// Enqueue plan + column scan + special rows for the candidates cands_d[0 .. *n_cand_d) (device memory; at most max_cands)
// of h's windows on the context's stream.  counts_d[c*4 + {perfect, F_mis, R_mis, trial}] are zeroed first when
// zero_counts is set.  bits_slot_d / bits_d: optional per-sequence bit vectors (device).  plans_ready: the caller has
// built the plans (and zeroed the counts) itself (mpb_cscan_plan.cuh).  No synchronisation.
int mpb_cscan_launch(mpb_hist* h, uint32_t fmask, uint32_t rmask, const mpb_cand* cands_d, const int* n_cand_d,
                     int max_cands, uint32_t* plans_d, unsigned long long* counts_d, int zero_counts,
                     const int32_t* bits_slot_d, uint32_t* bits_d, int plans_ready);

// The exhaustive pattern search behind mpb_pattern_hits (v < 0) and mpb_pattern_sites (v >= 0).  The hit outputs may be
// host or device memory (device: they stay there, as mpb_pattern_products needs); *n_hits may exceed max_hits.
// Synchronises the context's stream.
int mpb_pattern_search(mpb_msa* m, int32_t n_pat, const uint32_t* allow, const int32_t* lens, const uint32_t* strict,
                       int v, int64_t max_hits, int32_t* hit_pat, int32_t* hit_row, int32_t* hit_pos, int32_t* hit_mis,
                       int64_t* n_hits);
