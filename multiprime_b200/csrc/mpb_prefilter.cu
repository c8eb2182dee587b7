// mpb_prefilter.cu — entropy prefilter of the window pass on the column view, bit-sliced (SURVEY.md 8 a5; core:602-614, 723).
//
// What is computed: for every window a LOWER bound of the reference's total entropy tBit.  Every item the reference
// counts (each expansion of a cover row, each gap row) is mapped to a BS_BITS-bit code that is a function of the item's
// cells only; merging categories can only lower sum(-p log p), so the entropy of the code histogram bounds tBit from
// below, and a window whose bound is above the gate never needs a haplotype table.
//
// How: the row-domain kernel (k_prefilter in mpb200.cu) pays ~80 warp instructions per (window, 32 rows) and one global
// reduction per minority row — hundreds of millions of L2 reductions per pass on the 10^6 x 600 workload.  Here
//   * one CLUSTER of BS_CLUSTER thread blocks owns one window; each block keeps the window's whole histogram in shared
//     memory (8192 bins) for its share of the rows — no global atomics at all;
//   * a thread takes 32 sequences at a time (one word of the column view) and walks the window's k columns once: the row
//     classes of core:666-687 (edge gap, IUPAC cell -> special; the rest plain) are ORs / ANDs of plane words, and the
//     code is a GF(2)-linear hash — code bit i is the XOR of the low / high base bits of a fixed subset of the columns —
//     so all 32 codes come out bit-sliced from ~6 XORs per column;
//   * rows whose code equals the code of the window's reference k-mer (mpb_msa::cons) are counted with one popcount;
//     the others are transposed (13 x 32 bits -> 32 indices, SWAR) and counted with shared-memory atomics;
//   * special rows (0.6 % on the workload) are listed and handled at the end on the row view, expansion by expansion,
//     with the same code function evaluated by popcounts;
//   * the cluster's blocks then each sum their slice of the bins over all the cluster's histograms through distributed
//     shared memory and write (sum c, sum c log2 c) partials; the host adds the partials in rank order (deterministic).
// Algorithmic bytes: k/2 per (window, sequence) k-mer (SURVEY 8d); real traffic: 4 k plane words per (window, 32 rows)
// from L2, the column view itself (300 MB) from DRAM about once.
//
// Alignments with rows shorter than the alignment (unaligned input) keep the row-domain kernel.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "mpb200.h"
#include "mpb_host.h"
#include "mpb_device.cuh"
#include "mpb_prefilter.h"

namespace cg = cooperative_groups;

#define fail mpb_fail
#define CK MPB_CK

#define BS_BITS 13
#define BS_BINS (1 << BS_BITS)
#define BS_THREADS 256
#define BS_CLUSTER 8
#define BS_DEFER 2048

// per-column code patterns (weight 3, all 27 x {low, high, low ^ high} distinct): a difference in one cell always
// changes the code, and two single-cell differences never cancel
constexpr uint16_t BS_LO[27] = {0x414, 0x1900, 0x32, 0x13, 0xc40, 0xc4, 0x602, 0x1088, 0x4a0, 0xd, 0x1401, 0x409, 0x1a0, 0x248,
                                0x1204, 0x184, 0x100c, 0x1028, 0x1104, 0x1018, 0x58, 0x1006, 0x118, 0x881, 0xc8, 0x482, 0x504};
constexpr uint16_t BS_HI[27] = {0x608, 0x62, 0x1110, 0x811, 0x1802, 0xa04, 0x43, 0x320, 0x640, 0x86, 0x1a00, 0x40a, 0x809, 0x222,
                                0xa40, 0xe0, 0x806, 0x29, 0x1300, 0x501, 0x221, 0x841, 0x211, 0x1044, 0x460, 0x484, 0x920};
// the same patterns by code bit: mask over the columns whose low / high base bit enters code bit i
static __constant__ uint32_t c_bs_mlo[BS_BITS] = {0x800e08, 0x220004c, 0x425c221, 0x15b2a80, 0x58000d, 0x21104, 0x1102030,
                                                  0x38091a0, 0x4449002, 0x6040, 0x6000d51, 0x800012, 0x2f4482};
static __constant__ uint32_t c_bs_mhi[BS_BITS] = {0x7a1048, 0x12a52, 0x2810220, 0x21801, 0x40000c, 0x512a082, 0x1a0c142,
                                                  0x2008200, 0x40c0084, 0x5465a1, 0x3080901, 0x4215438, 0x840414};
static_assert(MPB_MAX_K <= 27, "code patterns cover 27 columns");

// code of one item given its one-hot planes (row view): gap cells count as base A
__device__ __forceinline__ uint32_t bs_code(uint32_t c, uint32_t g, uint32_t t) {
    const uint32_t lo = c | t, hi = g | t;
    uint32_t code = 0;
#pragma unroll
    for (int i = 0; i < BS_BITS; ++i) code |= ((__popc(lo & c_bs_mlo[i]) ^ __popc(hi & c_bs_mhi[i])) & 1u) << i;
    return code;
}

template <int J, int I>
__device__ __forceinline__ void bs_mix(uint32_t (&H)[16], uint32_t lo, uint32_t hi) {
    if constexpr (((BS_LO[J] >> I) & 1) != 0) H[I] ^= lo;
    if constexpr (((BS_HI[J] >> I) & 1) != 0) H[I] ^= hi;
    if constexpr (I + 1 < BS_BITS) bs_mix<J, I + 1>(H, lo, hi);
}

struct BsAcc {
    uint32_t anygap, allgap, anymul, gfirst, glast;
};

// columns J, J+1, ... k-1 of the window for word W of 32 sequences (q: plane A of column J, the same for all threads)
template <int J>
__device__ __forceinline__ void bs_cols(const uint32_t* __restrict__ q, long long nwords, unsigned W, int k, uint32_t (&H)[16],
                                        BsAcc& a) {
    if (J < k) {  // uniform
        const uint32_t A = __ldg(q + W), C = __ldg(q + nwords + W), G = __ldg(q + 2 * nwords + W), T = __ldg(q + 3 * nwords + W);
        const uint32_t gap = ~(A | C | G | T);
        a.anygap |= gap;
        a.allgap &= gap;
        a.anymul |= mpb_multi(A, C, G, T);
        if (J == 0) a.gfirst = gap;
        a.glast = gap;  // the last column walked is column k - 1
        bs_mix<J, 0>(H, C | T, G | T);
        if constexpr (J + 1 < MPB_MAX_K) bs_cols<J + 1>(q + 4 * nwords, nwords, W, k, H, a);
    }
}

#define BS_SWAP(i, j, m)                                      \
    {                                                         \
        const uint32_t t_ = ((H[i] >> (j)) ^ H[(i) + (j)]) & (m); \
        H[(i) + (j)] ^= t_;                                   \
        H[i] ^= t_ << (j);                                    \
    }

// one special row (edge gap / IUPAC / — never ragged here) on the row view: the items of core:666-711
__device__ __forceinline__ void bs_slow_row(const uint32_t* __restrict__ pl, int64_t nsp, int64_t s, int len, int p, int k,
                                            uint32_t kmask, int v, unsigned int* s_bins, int* __restrict__ err) {
    Win w;
    if (!mpb_load_window(pl, nsp, s, len, p, k, kmask, w)) atomicOr(err, MPB_ERR_SHORT_ROW);
    const bool isgap = __popc(w.gapv) > v;
    if (w.multi == 0 || isgap) {
        uint32_t c = w.c, g = w.g, tt = w.t;
        if (w.multi) {  // gap row holding IUPAC cells: one item, the lowest base of every cell
            const uint32_t a = w.a;
            c &= ~a;
            g &= ~(a | c);
            tt &= ~(a | c | g);
        }
        atomicAdd(&s_bins[bs_code(c, g, tt)], 1u);
    } else {
        const uint32_t total = mpb_expansions(w);
        if (total > MPB_MAX_EXP) {
            atomicOr(err, MPB_ERR_EXPAND);
        } else {
            for (uint32_t e = 0; e < total; ++e) {
                uint32_t a, c, g, tt;
                mpb_expand(w, e, a, c, g, tt);
                atomicAdd(&s_bins[bs_code(c, g, tt)], 1u);
            }
        }
    }
}

__global__ void __cluster_dims__(BS_CLUSTER, 1, 1) __launch_bounds__(BS_THREADS, 4)
k_prefilter_bs(const uint32_t* __restrict__ colp, long long nwords, const uint8_t* __restrict__ cons,
               const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq, const int32_t* __restrict__ lens, int k, int v,
               const int32_t* __restrict__ win_pos, double* __restrict__ part, int* __restrict__ err) {
    __shared__ unsigned int s_bins[BS_BINS];
    __shared__ unsigned int s_def[BS_DEFER];
    __shared__ unsigned int s_ndef;
    __shared__ unsigned int s_major;
    __shared__ double s_red[2][BS_THREADS / 32];
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned rank = cluster.block_rank();
    const int wi = blockIdx.x / BS_CLUSTER;
    const int p = win_pos[wi];
    const uint32_t kmask = (1u << k) - 1u;
    for (int i = threadIdx.x; i < BS_BINS; i += BS_THREADS) s_bins[i] = 0;
    if (threadIdx.x == 0) {
        s_ndef = 0;
        uint32_t lo = 0, hi = 0;  // the window's reference k-mer: the frequent base of every column
        for (int j = 0; j < k; ++j) {
            const uint32_t b = cons[p + j];
            lo |= (b & 1u) << j;
            hi |= ((b >> 1) & 1u) << j;
        }
        s_major = bs_code(lo & ~hi, hi & ~lo, lo & hi);
    }
    __syncthreads();
    const uint32_t major = s_major;
    const long long n_w = (n_seq + 31) / 32;
    const long long per = (n_w + BS_CLUSTER - 1) / BS_CLUSTER;
    const long long w_lo = (long long)rank * per, w_hi = (w_lo + per < n_w) ? w_lo + per : n_w;
    const uint32_t* __restrict__ col0 = colp + ((long long)p * 4) * nwords;
    unsigned my_count = 0;
    for (long long W = w_lo + threadIdx.x; W < w_hi; W += BS_THREADS) {
        const long long left = (long long)n_seq - W * 32;
        const uint32_t vm = left >= 32 ? 0xFFFFFFFFu : ((1u << left) - 1u);
        uint32_t H[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) H[i] = 0;
        BsAcc a = {0u, 0xFFFFFFFFu, 0u, 0u, 0u};
        bs_cols<0>(col0, nwords, (unsigned)W, k, H, a);
        const uint32_t special = ((a.gfirst | a.glast) & ~a.allgap) | a.anymul;
        const uint32_t plain = ~special & vm;
        uint32_t match = plain;
#pragma unroll
        for (int i = 0; i < BS_BITS; ++i) match &= ~(H[i] ^ (((major >> i) & 1u) ? 0xFFFFFFFFu : 0u));
        my_count += __popc(match);
        const uint32_t rest = plain & ~match;
        if (rest) {  // 13 x 32 bits -> one 13-bit index per sequence: word r = sequences r (low half) and r + 16 (high half)
            BS_SWAP(0, 8, 0x00FF00FFu) BS_SWAP(1, 8, 0x00FF00FFu) BS_SWAP(2, 8, 0x00FF00FFu) BS_SWAP(3, 8, 0x00FF00FFu)
            BS_SWAP(4, 8, 0x00FF00FFu) BS_SWAP(5, 8, 0x00FF00FFu) BS_SWAP(6, 8, 0x00FF00FFu) BS_SWAP(7, 8, 0x00FF00FFu)
            BS_SWAP(0, 4, 0x0F0F0F0Fu) BS_SWAP(1, 4, 0x0F0F0F0Fu) BS_SWAP(2, 4, 0x0F0F0F0Fu) BS_SWAP(3, 4, 0x0F0F0F0Fu)
            BS_SWAP(8, 4, 0x0F0F0F0Fu) BS_SWAP(9, 4, 0x0F0F0F0Fu) BS_SWAP(10, 4, 0x0F0F0F0Fu) BS_SWAP(11, 4, 0x0F0F0F0Fu)
            BS_SWAP(0, 2, 0x33333333u) BS_SWAP(1, 2, 0x33333333u) BS_SWAP(4, 2, 0x33333333u) BS_SWAP(5, 2, 0x33333333u)
            BS_SWAP(8, 2, 0x33333333u) BS_SWAP(9, 2, 0x33333333u) BS_SWAP(12, 2, 0x33333333u) BS_SWAP(13, 2, 0x33333333u)
            BS_SWAP(0, 1, 0x55555555u) BS_SWAP(2, 1, 0x55555555u) BS_SWAP(4, 1, 0x55555555u) BS_SWAP(6, 1, 0x55555555u)
            BS_SWAP(8, 1, 0x55555555u) BS_SWAP(10, 1, 0x55555555u) BS_SWAP(12, 1, 0x55555555u) BS_SWAP(14, 1, 0x55555555u)
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                if ((rest >> r) & 1u) atomicAdd(&s_bins[H[r] & 0xFFFFu], 1u);
                if ((rest >> (r + 16)) & 1u) atomicAdd(&s_bins[H[r] >> 16], 1u);
            }
        }
        uint32_t sp = special & vm;
        while (sp) {
            const int r = __ffs(sp) - 1;
            sp &= sp - 1;
            const int64_t s = W * 32 + r;
            const unsigned idx = atomicAdd(&s_ndef, 1u);
            if (idx < BS_DEFER) s_def[idx] = (unsigned)s;
            else bs_slow_row(pl, nsp, s, lens[s], p, k, kmask, v, s_bins, err);  // list full: where the row stands
        }
    }
    my_count = __reduce_add_sync(0xffffffffu, my_count);
    if ((threadIdx.x & 31) == 0 && my_count) atomicAdd(&s_bins[major], my_count);
    __syncthreads();
    const unsigned nd = s_ndef < BS_DEFER ? s_ndef : BS_DEFER;
    for (unsigned i = threadIdx.x; i < nd; i += BS_THREADS) {
        const int64_t s = (int64_t)s_def[i];
        bs_slow_row(pl, nsp, s, lens[s], p, k, kmask, v, s_bins, err);
    }
    cluster.sync();  // every block's histogram is complete
    const unsigned int* rb[BS_CLUSTER];
#pragma unroll
    for (int q = 0; q < BS_CLUSTER; ++q) rb[q] = cluster.map_shared_rank(s_bins, q);
    double a0 = 0, a1 = 0;
    const int slice = BS_BINS / BS_CLUSTER;
    for (int i = (int)rank * slice + threadIdx.x; i < ((int)rank + 1) * slice; i += BS_THREADS) {
        unsigned c = 0;
#pragma unroll
        for (int q = 0; q < BS_CLUSTER; ++q) c += rb[q][i];
        if (c) {
            a0 += (double)c;
            if (c > 1) a1 += (double)c * log2((double)c);
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    if ((threadIdx.x & 31) == 0) {
        s_red[0][threadIdx.x >> 5] = a0;
        s_red[1][threadIdx.x >> 5] = a1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < BS_THREADS / 32; ++w) {
            a0 += s_red[0][w];
            a1 += s_red[1][w];
        }
        part[((long long)wi * BS_CLUSTER + rank) * 2] = a0;
        part[((long long)wi * BS_CLUSTER + rank) * 2 + 1] = a1;
    }
    cluster.sync();  // nobody leaves while a peer still reads its histogram
}

int mpb_prefilter_bs(mpb_msa* m, int k, int v, const int32_t* win_pos, int32_t nw, double* s0_hd, double* s1_hd) {
    mpb_ctx* ctx = m->ctx;
    InBuf wp(ctx, win_pos, (size_t)nw * 4);
    if (wp.rc) return wp.rc;
    double* part = nullptr;
    CK(cudaMallocAsync(&part, (size_t)nw * BS_CLUSTER * 2 * sizeof(double), ctx->stream));
    ctx->pending_units = (double)nw * (double)m->n_seq;
    MPB_LAUNCH_NAMED(ctx, "k_prefilter", k_prefilter_bs, (unsigned)nw * BS_CLUSTER, BS_THREADS, 0, m->colp, (long long)m->nwords,
                     m->cons, m->planes, m->nsp, m->n_seq, m->lens, k, v, wp.dev<int32_t>(), part, m->err);
    std::vector<double> hp((size_t)nw * BS_CLUSTER * 2);
    CK(cudaMemcpyAsync(hp.data(), part, hp.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaFreeAsync(part, ctx->stream));
    int rc = mpb_check_flags(ctx, m->err);  // synchronises
    if (rc) return rc;
    const bool dev_out = mpb_is_device_ptr(s0_hd);
    std::vector<double> s0(nw), s1(nw);
    for (int w = 0; w < nw; ++w) {
        double a0 = 0, a1 = 0;
        for (int r = 0; r < BS_CLUSTER; ++r) {  // rank order: the same sums on every run
            a0 += hp[((size_t)w * BS_CLUSTER + r) * 2];
            a1 += hp[((size_t)w * BS_CLUSTER + r) * 2 + 1];
        }
        s0[w] = a0;
        s1[w] = a1;
    }
    if (dev_out) {
        CK(cudaMemcpyAsync(s0_hd, s0.data(), (size_t)nw * 8, cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(s1_hd, s1.data(), (size_t)nw * 8, cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    } else {
        memcpy(s0_hd, s0.data(), (size_t)nw * 8);
        memcpy(s1_hd, s1.data(), (size_t)nw * 8);
    }
    return 0;
}
