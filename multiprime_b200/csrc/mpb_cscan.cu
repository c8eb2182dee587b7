// mpb_cscan.cu — the candidate scan (mis_primer_check core:1103-1130, Y_distance core:229-233) on the COLUMN view of
// the alignment.
//
// Row kernel (k_scan, mpb200.cu): one thread = one sequence, ~90 warp instructions per candidate and 32 sequences.
// Here one thread = one candidate against the 32 sequences of a column-plane word:
//   * the mismatch word of primer position i is the complement of the OR of the allowed bases' plane words at column
//     p + i (a gap cell has no plane bit, so it always mismatches) — ONE coalesced 4-byte load for a plain position;
//   * mismatches are counted on the 32 lanes at once by a carry-save adder (three positions per step: 7 LOP3), with a
//     saturating top bit (variation <= 3: ones / twos / ">= 4");
//   * the 3'-end rules (core:1114-1127) are ORs of the mismatch words of the strict positions;
//   * counts are popcounts, reduced per warp and added with one atomic per warp, counter and candidate.
// About 90 warp instructions per candidate and 1024 sequences: a thirtieth of the row kernel's issue slots.
// Rows whose window is NOT the plain column cut (the window starts / ends inside a gap run and is patched with flank
// bases, holds IUPAC cells, or runs past a ragged row end: mpb_hist_build records them per window, with their patched
// windows) are masked out here and evaluated by k_cscan_special from the stored windows.
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "mpb200.h"
#include "mpb_host.h"
#include "mpb_device.cuh"
#include "mpb_cscan.h"
#include "mpb_cscan_plan.cuh"

#define fail mpb_fail
#define CK MPB_CK
#define LAUNCH MPB_LAUNCH

// ---- plans --------------------------------------------------------------------------------------------------------
// A plan turns a candidate into lists of column-plane rows (row = column * 4 + base):
//   hdr[0] n_tri   plain positions (one allowed base), three per step, padded with the all-ones row (never mismatches)
//   hdr[1] n_deg   entries of the degenerate positions (2..4 allowed bases each; bit 31 marks a position's last entry)
//   hdr[2] n_sf / hdr[3] n_sr   entries of the F- / R-strict positions (same format)
//   hdr[4] trial row or CSCAN_NONE, hdr[5] window index, hdr[6] offset of deg, hdr[7] offset of sf, sr follows
// tri region at word 8: [n_tri][4].
__global__ void k_cscan_plan(const mpb_cand* __restrict__ cands, const int* __restrict__ n_cand_ptr,
                             const int32_t* __restrict__ win_pos, int nw, int k, uint32_t fmask, uint32_t rmask,
                             uint32_t ones_row, uint32_t* __restrict__ plans, unsigned long long* __restrict__ counts,
                             int zero_counts, int* __restrict__ err) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= *n_cand_ptr) return;
    cscan_plan_one(c, cands, win_pos, nw, k, fmask, rmask, ones_row, plans, counts, zero_counts, err);
}

// ---- the column kernel ----------------------------------------------------------------------------------------------
// bit-sliced mismatch counter of 32 lanes; the top bit saturates
template <int NB>
struct Counter {
    uint32_t b[NB];
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int i = 0; i < NB; ++i) b[i] = 0;
    }
    // add a weight-2^from word
    __device__ __forceinline__ void add(uint32_t m, int from) {
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            if (i < from) continue;
            if (i == NB - 1) {
                b[i] |= m;
            } else {
                const uint32_t carry = b[i] & m;
                b[i] ^= m;
                m = carry;
            }
        }
    }
    // three weight-1 MATCH words (mismatch = complement): carry-save step
    __device__ __forceinline__ void add3(uint32_t x0, uint32_t x1, uint32_t x2) {
        const uint32_t s = ~(x0 ^ x1 ^ x2);                          // parity of the three mismatch bits
        const uint32_t c = ~((x0 & x1) | (x0 & x2) | (x1 & x2));     // at least two mismatches
        const uint32_t c1 = b[0] & s;
        b[0] ^= s;
        if (NB == 2) {
            b[1] |= c | c1;
        } else {
            const uint32_t t = b[1] ^ c ^ c1;
            const uint32_t c2 = (b[1] & c) | (b[1] & c1) | (c & c1);
            b[1] = t;
            add(c2, 2);
        }
    }
    // lanes whose count exceeds v (uniform)
    __device__ __forceinline__ uint32_t over(int v) const {
        uint32_t gt = 0, eq = 0xFFFFFFFFu;
#pragma unroll
        for (int i = NB - 1; i >= 0; --i) {
            const uint32_t vb = ((v >> i) & 1) ? 0xFFFFFFFFu : 0u;
            gt |= eq & b[i] & ~vb;
            eq &= ~(b[i] ^ vb);
        }
        return gt;
    }
    __device__ __forceinline__ uint32_t any() const {
        uint32_t a = 0;
#pragma unroll
        for (int i = 0; i < NB; ++i) a |= b[i];
        return a;
    }
};

#define CSCAN_THREADS 256
#define CSCAN_WPT 4  // words per thread: a block covers 1024 words = 32768 sequences per candidate

template <int NB, bool BITS>
__global__ void __launch_bounds__(CSCAN_THREADS)
k_cscan(const uint32_t* __restrict__ colp, long long nwords, int v, const uint32_t* __restrict__ plans,
        const int* __restrict__ n_cand_ptr, const uint32_t* __restrict__ spec_bits, const uint32_t* __restrict__ gap_bits,
        unsigned long long* __restrict__ counts, const int32_t* __restrict__ bits_slot, uint32_t* __restrict__ bits,
        long long out_words) {
    __shared__ __align__(16) uint32_t s_plan[CSCAN_THREADS / 32][CSCAN_PLAN_WORDS];
    const int n_cand = *n_cand_ptr;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* sp = s_plan[warp];
    const long long w0 = (long long)blockIdx.x * (CSCAN_THREADS * CSCAN_WPT) + threadIdx.x;
    const unsigned long long row_stride = (unsigned long long)(uint32_t)(nwords * 4);  // bytes per column-plane row (< 2^28)
    for (int c = blockIdx.y; c < n_cand; c += gridDim.y) {
        const uint32_t* P = plans + (size_t)c * CSCAN_PLAN_WORDS;
        __syncwarp();
        const uint32_t used = __ldg(P + 7) + __ldg(P + 2) + __ldg(P + 3);
        for (uint32_t i = lane; i < used; i += 32) sp[i] = __ldg(P + i);
        __syncwarp();
        const int ntri = (int)sp[0], nd = (int)sp[1], nsf = (int)sp[2], nsr = (int)sp[3];
        const uint32_t trial = sp[4];
        const int win = (int)sp[5];
        const uint32_t* pdeg = sp + sp[6];
        const uint32_t* psf = sp + sp[7];
        const uint32_t* psr = psf + nsf;
        unsigned n0 = 0, nf = 0, nr = 0, nt = 0;
        // two words per pass: their plane loads are independent, so twice as many are in flight per thread
#pragma unroll 1
        for (int j = 0; j < CSCAN_WPT; j += 2) {
            const long long wa = w0 + (long long)j * CSCAN_THREADS;
            if (wa >= nwords) break;
            long long wb = wa + CSCAN_THREADS;
            const bool two = wb < nwords;
            if (!two) wb = wa;  // (re-reads word a; its results are dropped)
            const char* base_a = reinterpret_cast<const char*>(colp + wa);
            const char* base_b = reinterpret_cast<const char*>(colp + wb);
#define LD_A(row) __ldg(reinterpret_cast<const uint32_t*>(base_a + (row) * row_stride))
#define LD_B(row) __ldg(reinterpret_cast<const uint32_t*>(base_b + (row) * row_stride))
            Counter<NB> ca, cb;
            ca.clear();
            cb.clear();
            for (int t = 0; t < ntri; ++t) {
                const uint4 r = *reinterpret_cast<const uint4*>(sp + 8 + 4 * t);
                const uint32_t a0 = LD_A(r.x), a1 = LD_A(r.y), a2 = LD_A(r.z);
                const uint32_t b0 = LD_B(r.x), b1 = LD_B(r.y), b2 = LD_B(r.z);
                ca.add3(a0, a1, a2);
                cb.add3(b0, b1, b2);
            }
            {
                uint32_t xa = 0, xb = 0;
                for (int e = 0; e < nd; ++e) {
                    const uint32_t r = pdeg[e];
                    xa |= LD_A(r & 0x7FFFFFFFu);
                    xb |= LD_B(r & 0x7FFFFFFFu);
                    if (r >> 31) {
                        ca.add(~xa, 0);
                        cb.add(~xb, 0);
                        xa = xb = 0;
                    }
                }
            }
            uint32_t mfa = 0, mra = 0, mfb = 0, mrb = 0;
            {
                uint32_t xa = 0, xb = 0;
                for (int e = 0; e < nsf; ++e) {
                    const uint32_t r = psf[e];
                    xa |= LD_A(r & 0x7FFFFFFFu);
                    xb |= LD_B(r & 0x7FFFFFFFu);
                    if (r >> 31) {
                        mfa |= ~xa;
                        mfb |= ~xb;
                        xa = xb = 0;
                    }
                }
                for (int e = 0; e < nsr; ++e) {
                    const uint32_t r = psr[e];
                    xa |= LD_A(r & 0x7FFFFFFFu);
                    xb |= LD_B(r & 0x7FFFFFFFu);
                    if (r >> 31) {
                        mra |= ~xa;
                        mrb |= ~xb;
                        xa = xb = 0;
                    }
                }
            }
            const uint32_t spec_a = __ldg(spec_bits + (long long)win * nwords + wa);
            const uint32_t spec_b = two ? __ldg(spec_bits + (long long)win * nwords + wb) : 0xFFFFFFFFu;
            const uint32_t over_a = ca.over(v), over_b = cb.over(v);
            const uint32_t perf_a = ~ca.any() & ~spec_a, perf_b = ~cb.any() & ~spec_b;
            n0 += __popc(perf_a) + __popc(perf_b);
            nf += __popc(~(over_a | mfa | spec_a)) + __popc(~(over_b | mfb | spec_b));
            nr += __popc(~(over_a | mra | spec_a)) + __popc(~(over_b | mrb | spec_b));
            if (trial != CSCAN_NONE) nt += __popc(perf_a & LD_A(trial)) + __popc(perf_b & LD_B(trial));
            if (BITS) {
                const int slot = bits_slot[c];
                if (slot >= 0) {
                    uint32_t* o = bits + (long long)slot * 3 * out_words;
                    if (wa < out_words) {
                        const uint32_t gapw = __ldg(gap_bits + (long long)win * nwords + wa);
                        o[wa] = (over_a | mfa) & ~spec_a & ~gapw;   // gap rows carry no non-cover bit (core:689-698)
                        o[out_words + wa] = (over_a | mra) & ~spec_a & ~gapw;
                        o[2 * out_words + wa] = gapw;
                    }
                    if (two && wb < out_words) {
                        const uint32_t gapw = __ldg(gap_bits + (long long)win * nwords + wb);
                        o[wb] = (over_b | mfb) & ~spec_b & ~gapw;
                        o[out_words + wb] = (over_b | mrb) & ~spec_b & ~gapw;
                        o[2 * out_words + wb] = gapw;
                    }
                }
            }
#undef LD_A
#undef LD_B
        }
        n0 = __reduce_add_sync(0xffffffffu, n0);
        nf = __reduce_add_sync(0xffffffffu, nf);
        nr = __reduce_add_sync(0xffffffffu, nr);
        nt = __reduce_add_sync(0xffffffffu, nt);
        if (lane < 4) {
            const unsigned val = lane == 0 ? n0 : (lane == 1 ? nf - n0 : (lane == 2 ? nr - n0 : nt));
            if (val) atomicAdd(&counts[(size_t)c * 4 + lane], (unsigned long long)val);
        }
    }
}

// ---- the special rows: one block per candidate walks the stored windows of the candidate's window -----------------
template <bool BITS>
__global__ void __launch_bounds__(256)
k_cscan_special(const mpb_cand* __restrict__ cands, const int* __restrict__ n_cand_ptr, int nw, int k, int v, uint32_t fmask,
                uint32_t rmask, const uint4* __restrict__ spec_win, const int32_t* __restrict__ spec_row,
                const unsigned long long* __restrict__ spec_n, long long spec_cap, unsigned long long* __restrict__ counts,
                const int32_t* __restrict__ bits_slot, uint32_t* __restrict__ bits, long long out_words,
                int* __restrict__ err) {
    __shared__ unsigned s_acc[4];
    const int n_cand = *n_cand_ptr;
    const uint32_t kmask = (1u << k) - 1u;
    for (int c = blockIdx.x; c < n_cand; c += gridDim.x) {
        const mpb_cand cd = cands[c];
        if (cd.win < 0 || cd.win >= nw) continue;
        long long n = (long long)spec_n[cd.win];
        if (n > spec_cap) n = spec_cap;
        if ((long long)blockIdx.y * 256 >= n) continue;  // uniform: this slice of the list is empty
        if (threadIdx.x < 4) s_acc[threadIdx.x] = 0;
        __syncthreads();
        const uint32_t nA = ~cd.allow[0] & kmask, nC = ~cd.allow[1] & kmask, nG = ~cd.allow[2] & kmask, nT = ~cd.allow[3] & kmask;
        const int tpos = cd.trial >= 0 ? (cd.trial & 255) : 0, tbase = cd.trial >= 0 ? ((cd.trial >> 8) & 3) : -1;
        unsigned n0 = 0, nf = 0, nr = 0, nt = 0;
        for (long long i = (long long)blockIdx.y * 256 + threadIdx.x; i < n; i += 256ll * gridDim.y) {
            const uint4 q = __ldg(spec_win + (long long)cd.win * spec_cap + i);
            Win w;
            w.a = q.x;
            w.c = q.y;
            w.g = q.z;
            w.t = q.w;
            w.gapv = ~(q.x | q.y | q.z | q.w) & kmask;
            w.multi = mpb_multi(q.x, q.y, q.z, q.w);
            uint32_t nexp = 1;
            if (w.multi) {
                nexp = mpb_expansions(w);
                if (nexp > MPB_MAX_EXP) {
                    atomicOr(err, MPB_ERR_EXPAND);
                    continue;
                }
            }
            bool nonf = false, nonr = false;
            for (uint32_t x = 0; x < nexp; ++x) {
                uint32_t a = w.a, cc = w.c, g = w.g, tt = w.t;
                if (w.multi) mpb_expand(w, x, a, cc, g, tt);
                const uint32_t mis = w.gapv | (a & nA) | (cc & nC) | (g & nG) | (tt & nT);
                const bool within = __popc(mis) <= v;
                const bool z = mis == 0u;
                const bool okf = within && (mis & fmask) == 0u, okr = within && (mis & rmask) == 0u;
                n0 += z;
                nf += okf && !z;
                nr += okr && !z;
                if (tbase >= 0 && z) {
                    const uint32_t pl = tbase == 0 ? a : (tbase == 1 ? cc : (tbase == 2 ? g : tt));
                    nt += (pl >> tpos) & 1u;
                }
                nonf |= !okf;
                nonr |= !okr;
            }
            if (BITS) {
                const int slot = bits_slot[c];
                if (slot >= 0) {
                    const int s = spec_row[(long long)cd.win * spec_cap + i];
                    uint32_t* o = bits + (long long)slot * 3 * out_words;
                    if (nonf) atomicOr(&o[s >> 5], 1u << (s & 31));
                    if (nonr) atomicOr(&o[out_words + (s >> 5)], 1u << (s & 31));
                }
            }
        }
        n0 = __reduce_add_sync(0xffffffffu, n0);
        nf = __reduce_add_sync(0xffffffffu, nf);
        nr = __reduce_add_sync(0xffffffffu, nr);
        nt = __reduce_add_sync(0xffffffffu, nt);
        if ((threadIdx.x & 31) == 0) {
            if (n0) atomicAdd(&s_acc[0], n0);
            if (nf) atomicAdd(&s_acc[1], nf);
            if (nr) atomicAdd(&s_acc[2], nr);
            if (nt) atomicAdd(&s_acc[3], nt);
        }
        __syncthreads();
        if (threadIdx.x < 4 && s_acc[threadIdx.x]) atomicAdd(&counts[(size_t)c * 4 + threadIdx.x], (unsigned long long)s_acc[threadIdx.x]);
        __syncthreads();
    }
}

// ---- launch helper shared with the device walk ------------------------------------------------------------------------
int mpb_cscan_launch(mpb_hist* h, uint32_t fmask, uint32_t rmask, const mpb_cand* cands_d, const int* n_cand_d,
                     int max_cands, uint32_t* plans_d, unsigned long long* counts_d, int zero_counts,
                     const int32_t* bits_slot_d, uint32_t* bits_d, int plans_ready) {
    mpb_msa* m = h->msa;
    mpb_ctx* ctx = m->ctx;
    if (h->v > 15) return fail(MPB_EINVAL, "the column scan supports variation <= 15 (got %d)", h->v);
    if (!h->spec_bits || !h->spec_win) return fail(MPB_EINVAL, "this mpb_hist was not built from the alignment (no row classes)");
    if (max_cands < 1) return 0;
    if (!plans_ready)
        LAUNCH(ctx, k_cscan_plan, (unsigned)((max_cands + 127) / 128), 128, 0, cands_d, n_cand_d, h->win_pos, h->nw, h->k, fmask,
               rmask, MPB_COLP_ONES(m), plans_d, counts_d, zero_counts, m->err);
    const long long per_block = (long long)CSCAN_THREADS * CSCAN_WPT;
    const unsigned gx = (unsigned)((m->nwords + per_block - 1) / per_block);
    unsigned gy = (unsigned)(((long long)ctx->sm_count * 8 + gx - 1) / gx);
    if (gy > (unsigned)max_cands) gy = (unsigned)max_cands;
    if (gy < 1) gy = 1;
    const long long out_words = (m->n_seq + 31) / 32;
    // special rows: blocks (candidate, slice of the window's list); enough slices that a list of spec_cap rows is walked
    // in a few iterations
    unsigned spec_gy = (unsigned)((h->spec_cap + 256 * 4 - 1) / (256 * 4));
    if (spec_gy < 1) spec_gy = 1;
    if (spec_gy > 16) spec_gy = 16;
    if (bits_slot_d) {
        if (h->v <= 3)
            MPB_LAUNCH_NAMED(ctx, "k_cscan", (k_cscan<3, true>), dim3(gx, gy), CSCAN_THREADS, 0, m->colp, (long long)m->nwords, h->v, plans_d,
                   n_cand_d, h->spec_bits, h->gap_bits, counts_d, bits_slot_d, bits_d, out_words);
        else
            MPB_LAUNCH_NAMED(ctx, "k_cscan", (k_cscan<5, true>), dim3(gx, gy), CSCAN_THREADS, 0, m->colp, (long long)m->nwords, h->v, plans_d,
                   n_cand_d, h->spec_bits, h->gap_bits, counts_d, bits_slot_d, bits_d, out_words);
        MPB_LAUNCH_NAMED(ctx, "k_cscan_special", k_cscan_special<true>, dim3((unsigned)(max_cands < 4096 ? max_cands : 4096), spec_gy), 256, 0, cands_d, n_cand_d, h->nw,
               h->k, h->v, fmask, rmask, h->spec_win, h->spec_row, h->spec_n, (long long)h->spec_cap, counts_d, bits_slot_d,
               bits_d, out_words, m->err);
    } else {
        if (h->v <= 3)
            MPB_LAUNCH_NAMED(ctx, "k_cscan", (k_cscan<3, false>), dim3(gx, gy), CSCAN_THREADS, 0, m->colp, (long long)m->nwords, h->v, plans_d,
                   n_cand_d, h->spec_bits, h->gap_bits, counts_d, (const int32_t*)nullptr, (uint32_t*)nullptr, out_words);
        else
            MPB_LAUNCH_NAMED(ctx, "k_cscan", (k_cscan<5, false>), dim3(gx, gy), CSCAN_THREADS, 0, m->colp, (long long)m->nwords, h->v, plans_d,
                   n_cand_d, h->spec_bits, h->gap_bits, counts_d, (const int32_t*)nullptr, (uint32_t*)nullptr, out_words);
        MPB_LAUNCH_NAMED(ctx, "k_cscan_special", k_cscan_special<false>, dim3((unsigned)(max_cands < 4096 ? max_cands : 4096), spec_gy), 256, 0, cands_d, n_cand_d, h->nw,
               h->k, h->v, fmask, rmask, h->spec_win, h->spec_row, h->spec_n, (long long)h->spec_cap, counts_d,
               (const int32_t*)nullptr, (uint32_t*)nullptr, out_words, m->err);
    }
    return 0;
}

extern "C" int mpb_cscan(mpb_hist* h, uint32_t fmask, uint32_t rmask, const mpb_cand* cands_hd, int64_t nc,
                         int64_t* counts_hd, const int32_t* bits_slot, uint32_t* bits_hd) {
    if (!h || !cands_hd || !counts_hd) return fail(MPB_EINVAL, "NULL argument");
    if (nc < 1) return 0;
    if (nc >= (1ll << 24)) return fail(MPB_EINVAL, "too many candidates in one call");
    if (bits_slot && !bits_hd) return fail(MPB_EINVAL, "bits_slot without bits");
    mpb_msa* m = h->msa;
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    const long long out_words = (m->n_seq + 31) / 32;
    int nslots = 0;
    if (bits_slot)
        for (int64_t i = 0; i < nc; ++i)
            if (bits_slot[i] >= nslots) nslots = bits_slot[i] + 1;
    InBuf ca(ctx, cands_hd, (size_t)nc * sizeof(mpb_cand)), bs(ctx, bits_slot, (size_t)nc * 4);
    OutBuf oc(ctx, counts_hd, (size_t)nc * 4 * 8), ob(ctx, bits_hd, (size_t)nslots * 3 * out_words * 4);
    if (ca.rc || bs.rc || oc.rc || ob.rc) return MPB_ECUDA;
    uint32_t* plans = nullptr;
    int* n_d = nullptr;
    CK(cudaMallocAsync(&plans, (size_t)nc * CSCAN_PLAN_WORDS * 4, ctx->stream));
    CK(cudaMallocAsync(&n_d, 4, ctx->stream));
    const int n32 = (int)nc;
    CK(cudaMemcpyAsync(n_d, &n32, 4, cudaMemcpyHostToDevice, ctx->stream));
    ctx->pending_units = 0;
    ctx->extra_units["k_cscan"] += (double)nc * (double)m->n_seq;
    int rc = mpb_cscan_launch(h, fmask, rmask, ca.dev<mpb_cand>(), n_d, n32, plans, oc.dev<unsigned long long>(), 1,
                              bits_slot ? bs.dev<int32_t>() : nullptr, ob.dev<uint32_t>(), 0);
    CK(cudaFreeAsync(plans, ctx->stream));
    CK(cudaFreeAsync(n_d, ctx->stream));
    if (rc) return rc;
    CK(oc.finish());
    CK(ob.finish());
    return mpb_check_flags(ctx, m->err);  // synchronises: host staging buffers and n32 stay alive until here
}

// ---- exhaustive pattern search (SURVEY.md 8f-4) -----------------------------------------------------------------------
// Every position of every sequence against a set of degenerate patterns: the in-silico PCR of
// extract_PCR_product_V1.py:189-216 and primer_coverage.py asks "where does an expansion of this primer occur (with at
// most v mismatches) in this sequence".  On the column view that is the scan kernel with the window start as a free
// variable: thread = (position, 32-sequence word).  Sites are rare and leave as (pattern, sequence, position[,
// mismatches]) tuples.  A cell matches only when it holds exactly one base and that base is allowed: an IUPAC cell sets
// two or more planes and the reference's plain-text search never matches it.  Columns are walked with stride gridDim.y
// (capped at 65535), so lines of any width fit one launch.
//   NB == 0  exact search (mpb_pattern_hits): the running AND of the per-column match words dies after two or three
//            columns almost everywhere.
//   NB > 0   mismatch-bounded search (mpb_pattern_sites): per-lane mismatch counts in NB bit-sliced saturating words (the
//            Counter of k_cscan), the mismatch words of the strict positions ORed into a "dead" word; a lane stops when
//            it is dead or over v, so on random sequence the walk ends after about v + 2 columns.  Cells past a row's
//            length are zero (no base) and no longer rule a site out, so emitted sites are checked against lens.
struct mpb_pattern {
    uint32_t allow[4];
    int32_t len;
    uint32_t strict;  // positions where a mismatch disqualifies the site (NB > 0 only)
};

#define PATTERN_MAX_GY 65535

template <int NB>
__global__ void __launch_bounds__(256)
k_pattern_hits(const uint32_t* __restrict__ colp, long long nwords, int n_col, const mpb_pattern* __restrict__ pats, int n_pat,
               int v, long long n_seq, const int32_t* __restrict__ lens, long long max_hits, int32_t* __restrict__ hit_pat,
               int32_t* __restrict__ hit_row, int32_t* __restrict__ hit_pos, int32_t* __restrict__ hit_mis,
               unsigned long long* __restrict__ n_hits) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwords) return;
    for (int x = blockIdx.y; x < n_col; x += gridDim.y) {
        for (int p = 0; p < n_pat; ++p) {
            const mpb_pattern pt = pats[p];
            if (x + pt.len > n_col) continue;
            uint32_t acc = 0xFFFFFFFFu;  // NB == 0: lanes still matching; NB > 0: lanes neither dead nor over v
            Counter<NB == 0 ? 1 : NB> cnt;
            cnt.clear();
            uint32_t dead = 0;
            for (int i = 0; i < pt.len && acc; ++i) {
                const uint32_t* c = colp + (long long)(x + i) * 4 * nwords + w;
                const uint32_t pa = __ldg(c), pc = __ldg(c + nwords), pg = __ldg(c + 2 * nwords), pt4 = __ldg(c + 3 * nwords);
                const uint32_t multi = ((pa | pc) & (pg | pt4)) | (pa & pc) | (pg & pt4);  // two or more planes set
                uint32_t m = 0;
                if ((pt.allow[0] >> i) & 1u) m |= pa;
                if ((pt.allow[1] >> i) & 1u) m |= pc;
                if ((pt.allow[2] >> i) & 1u) m |= pg;
                if ((pt.allow[3] >> i) & 1u) m |= pt4;
                if (NB == 0) {
                    acc &= m & ~multi;
                } else {
                    const uint32_t mis = ~(m & ~multi);
                    if ((pt.strict >> i) & 1u) dead |= mis;
                    cnt.add(mis, 0);
                    acc = ~(dead | cnt.over(v));
                }
            }
            while (acc) {
                const int bit = __ffs(acc) - 1;
                acc &= acc - 1;
                const long long row = w * 32 + bit;
                if (NB > 0 && (row >= n_seq || x + pt.len > __ldg(lens + row))) continue;
                const unsigned long long slot = atomicAdd(n_hits, 1ull);
                if ((long long)slot < max_hits) {
                    hit_pat[slot] = p;
                    hit_row[slot] = (int32_t)row;
                    hit_pos[slot] = x;
                    if (NB > 0) {
                        int nm = 0;
#pragma unroll
                        for (int b = 0; b < (NB == 0 ? 1 : NB); ++b) nm |= (int)((cnt.b[b] >> bit) & 1u) << b;
                        hit_mis[slot] = nm;
                    }
                }
            }
        }
    }
}

// v < 0: exact search (mpb_pattern_hits; strict and hit_mis unused)
int mpb_pattern_search(mpb_msa* m, int32_t n_pat, const uint32_t* allow, const int32_t* lens, const uint32_t* strict,
                       int v, int64_t max_hits, int32_t* hit_pat, int32_t* hit_row, int32_t* hit_pos, int32_t* hit_mis,
                       int64_t* n_hits) {
    if (!m || !allow || !lens || !hit_pat || !hit_row || !hit_pos || !n_hits) return fail(MPB_EINVAL, "NULL argument");
    if (v >= 0 && (!strict || !hit_mis)) return fail(MPB_EINVAL, "NULL argument");
    if (n_pat < 1 || max_hits < 0) return fail(MPB_EINVAL, "bad n_pat or max_hits");
    if (v > 15) return fail(MPB_EINVAL, "at most 15 mismatches are supported (got %d)", v);
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::vector<mpb_pattern> pats(n_pat);
    for (int i = 0; i < n_pat; ++i) {
        if (lens[i] < 1 || lens[i] > 32) return fail(MPB_EINVAL, "pattern %d: length %d outside 1..32", i, lens[i]);
        if (v >= lens[i])
            return fail(MPB_EINVAL, "pattern %d: %d mismatches allowed on a %d-base pattern match everywhere", i, v, lens[i]);
        for (int b = 0; b < 4; ++b) pats[i].allow[b] = allow[i * 4 + b];
        pats[i].len = lens[i];
        pats[i].strict = v >= 0 ? strict[i] : 0u;
    }
    InBuf pd(ctx, pats.data(), pats.size() * sizeof(mpb_pattern));
    OutBuf op(ctx, hit_pat, (size_t)max_hits * 4), orow(ctx, hit_row, (size_t)max_hits * 4), opos(ctx, hit_pos, (size_t)max_hits * 4),
        omis(ctx, v >= 0 ? hit_mis : nullptr, v >= 0 ? (size_t)max_hits * 4 : 0);
    if (pd.rc || op.rc || orow.rc || opos.rc || omis.rc) return MPB_ECUDA;
    unsigned long long* dn = nullptr;
    CK(cudaMallocAsync(&dn, 8, ctx->stream));
    CK(cudaMemsetAsync(dn, 0, 8, ctx->stream));
    ctx->pending_units = (double)n_pat * (double)m->n_seq * (double)m->n_col;
    const unsigned gy = (unsigned)(m->n_col < PATTERN_MAX_GY ? m->n_col : PATTERN_MAX_GY);
    const dim3 grid((unsigned)((m->nwords + 255) / 256), gy);
#define PATTERN_ARGS                                                                                                       \
    m->colp, (long long)m->nwords, (int)m->n_col, pd.dev<mpb_pattern>(), (int)n_pat, v, (long long)m->n_seq, m->lens,      \
        (long long)max_hits, op.dev<int32_t>(), orow.dev<int32_t>(), opos.dev<int32_t>(), omis.dev<int32_t>(), dn
    if (v < 0)
        MPB_LAUNCH_NAMED(ctx, "k_pattern_hits", k_pattern_hits<0>, grid, 256, 0, PATTERN_ARGS);
    else if (v <= 3)
        MPB_LAUNCH_NAMED(ctx, "k_pattern_sites", k_pattern_hits<3>, grid, 256, 0, PATTERN_ARGS);
    else
        MPB_LAUNCH_NAMED(ctx, "k_pattern_sites", k_pattern_hits<5>, grid, 256, 0, PATTERN_ARGS);
#undef PATTERN_ARGS
    unsigned long long n = 0;
    CK(cudaMemcpyAsync(&n, dn, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(op.finish());
    CK(orow.finish());
    CK(opos.finish());
    CK(omis.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaFreeAsync(dn, ctx->stream));
    *n_hits = (int64_t)n;
    return 0;
}

extern "C" int mpb_pattern_hits(mpb_msa* m, int32_t n_pat, const uint32_t* allow, const int32_t* lens, int64_t max_hits,
                                int32_t* hit_pat, int32_t* hit_row, int32_t* hit_pos, int64_t* n_hits) {
    return mpb_pattern_search(m, n_pat, allow, lens, nullptr, -1, max_hits, hit_pat, hit_row, hit_pos, nullptr, n_hits);
}

extern "C" int mpb_pattern_sites(mpb_msa* m, int32_t n_pat, const uint32_t* allow, const int32_t* lens,
                                 const uint32_t* strict, int32_t v, int64_t max_hits, int32_t* hit_pat, int32_t* hit_row,
                                 int32_t* hit_pos, int32_t* hit_mis, int64_t* n_hits) {
    if (v < 0) return fail(MPB_EINVAL, "negative mismatch bound %d", v);
    return mpb_pattern_search(m, n_pat, allow, lens, strict, v, max_hits, hit_pat, hit_row, hit_pos, hit_mis, n_hits);
}
