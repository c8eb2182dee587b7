// mpb_products.cu — in-silico PCR over every primer combination of a set (mpb_pattern_products; primer_specificity.py).
//
// The sites of mpb_pattern_sites never leave HBM:
//   search   k_pattern_sites into device buffers (grown and re-run when the count overflows);
//   filter   k_products_filter maps (row, x) to the stream, drops sites at x >= S (the next row owns them) and sites that
//            leave their record, and splits them into left and right sites, each packed into one 64-bit sort key:
//              left  = primer << 47 | stream position << 4 | mismatches
//              right = stream position << 14 | primer << 4 | mismatches
//   sort     cub::DeviceRadixSort of both lists: left sites fall into runs of one (primer, record), right sites are in
//            stream order;
//   segments a run cut into pieces of at most PROD_SEG sites (and at the chunk budget) is one join block;
//   join     k_products_join: every thread takes one left site, finds its right-site window by binary search and adds
//            its products to per-right-primer accumulators in shared memory (a 64-bit count and the best product as
//            one packed integer merged with atomicMin); the block emits one partial group per right primer it saw;
//   reduce   partial groups are sorted by (record, i, j) and merged (sum of counts, min of best) per chunk of left sites,
//            and once more over the chunks: device memory is bounded by sites + groups, never by products, and the
//            merge is associative and commutative, so the result does not depend on launch order;
//   summary  per-combination products / targets / perfect targets, the per-record union of the listed combinations,
//            and the listed groups in (record, i, j) order (DeviceScan of the listed flags).
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "mpb200.h"
#include "mpb_cscan.h"
#include "mpb_host.h"

#define fail mpb_fail
#define CK MPB_CK

#define PROD_SEG 128                      // left sites per join block
#define PROD_MAX_PRIMERS 1024             // 10 bits of primer index in the keys
#define PROD_POS_BITS 43                  // stream positions of one handle
#define PROD_MAX_HI ((1 << 23) - 1)       // 23 bits of product length in the packed best
#define PROD_MAX_RECORD 0xFFFFFFFFll      // 32 bits of start in the packed best
#define PROD_CHUNK (1ll << 22)            // default left sites per join pass

// best product of a group, smallest first: total mismatches (5 bits) | length (23) | start (32) | left mismatches (4).
// The left mismatches follow from (i, start), so they never decide the order.
__device__ __forceinline__ unsigned long long pack_best(int tot, long long len, long long start, int lmis) {
    return ((unsigned long long)tot << 59) | ((unsigned long long)len << 36) | ((unsigned long long)start << 4) |
           (unsigned long long)lmis;
}

struct ProdAcc {
    unsigned long long cnt, best;
};
struct ProdMerge {
    __host__ __device__ ProdAcc operator()(const ProdAcc& a, const ProdAcc& b) const {
        return ProdAcc{a.cnt + b.cnt, a.best < b.best ? a.best : b.best};
    }
};

__device__ __forceinline__ int find_record(const int64_t* __restrict__ off, int n_rec, long long g) {
    int lo = 0, hi = n_rec;  // last record starting at or before g
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(off + mid) <= g) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

__global__ void k_products_filter(const int32_t* __restrict__ hp, const int32_t* __restrict__ hr,
                                  const int32_t* __restrict__ hx, const int32_t* __restrict__ hm, long long n,
                                  const int32_t* __restrict__ pat_primer, const int32_t* __restrict__ pat_side,
                                  const int32_t* __restrict__ pat_len, long long stride, const int64_t* __restrict__ off,
                                  const int64_t* __restrict__ len, int n_rec, unsigned long long* __restrict__ lkey,
                                  unsigned long long* __restrict__ rkey, unsigned long long* __restrict__ n_lr) {
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const long long x = hx[k];
        if (x >= stride) continue;
        const long long g = (long long)hr[k] * stride + x;
        const int r = find_record(off, n_rec, g);
        if (r < 0) continue;
        const int p = hp[k];
        if (g + __ldg(pat_len + p) > __ldg(off + r) + __ldg(len + r)) continue;
        const unsigned long long prim = (unsigned long long)__ldg(pat_primer + p), mis = (unsigned long long)hm[k];
        if (__ldg(pat_side + p) == 0) {
            const unsigned long long slot = atomicAdd(n_lr, 1ull);
            lkey[slot] = prim << 47 | (unsigned long long)g << 4 | mis;
        } else {
            const unsigned long long slot = atomicAdd(n_lr + 1, 1ull);
            rkey[slot] = (unsigned long long)g << 14 | prim << 4 | mis;
        }
    }
}

// head[k] = 1 where a join segment starts: a new (primer, record) run, or every seg_len sites of the list
__global__ void k_products_heads(const unsigned long long* __restrict__ lkey, long long n, const int64_t* __restrict__ off,
                                 int n_rec, int seg_len, int32_t* __restrict__ lrec, uint32_t* __restrict__ head) {
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const unsigned long long key = lkey[k];
        const int r = find_record(off, n_rec, (long long)((key >> 4) & ((1ull << PROD_POS_BITS) - 1)));
        lrec[k] = r;
        bool h = k == 0 || k % seg_len == 0;
        if (!h) {
            const unsigned long long prev = lkey[k - 1];
            h = (prev >> 47) != (key >> 47) ||
                find_record(off, n_rec, (long long)((prev >> 4) & ((1ull << PROD_POS_BITS) - 1))) != r;
        }
        head[k] = h;
    }
}

__global__ void k_products_segments(const uint32_t* __restrict__ head, const uint32_t* __restrict__ pos, long long n,
                                    int32_t* __restrict__ seg_start) {
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        if (head[k]) seg_start[pos[k]] = (int32_t)k;
        if (k == n - 1) seg_start[pos[k] + head[k]] = (int32_t)n;
    }
}

__global__ void __launch_bounds__(PROD_SEG)
k_products_join(const unsigned long long* __restrict__ lkey, const int32_t* __restrict__ lrec,
                const int32_t* __restrict__ seg_start, long long seg0, const unsigned long long* __restrict__ rkey,
                long long n_right, const int32_t* __restrict__ plen, int n_primer, int lmin, int lmax, int lo, int hi,
                const int64_t* __restrict__ off, const int64_t* __restrict__ len, unsigned long long* __restrict__ pkey,
                ProdAcc* __restrict__ pacc, unsigned long long* __restrict__ n_part, long long cap) {
    extern __shared__ unsigned long long sh[];
    unsigned long long* cnt = sh;
    unsigned long long* best = sh + n_primer;
    for (int j = threadIdx.x; j < n_primer; j += blockDim.x) {
        cnt[j] = 0;
        best[j] = ~0ull;
    }
    __syncthreads();
    const long long s = seg0 + blockIdx.x;
    const long long a = seg_start[s], b = seg_start[s + 1];
    const long long k = a + threadIdx.x;
    if (k < b) {
        const unsigned long long key = lkey[k];
        const int i = (int)(key >> 47), lm = (int)(key & 15);
        const long long g = (long long)((key >> 4) & ((1ull << PROD_POS_BITS) - 1));
        const int r = lrec[k];
        const long long o = __ldg(off + r), end = o + __ldg(len + r);
        const int li = __ldg(plen + i);
        const long long ylo = g + max(li, lo - lmax);
        const long long yhi = min(g + hi - lmin, end - lmin);
        long long q0 = 0, q1 = n_right;  // first right site at or after ylo
        const unsigned long long want = (unsigned long long)ylo << 14;
        while (q0 < q1) {
            const long long mid = (q0 + q1) >> 1;
            if (__ldg(rkey + mid) < want) q0 = mid + 1;
            else q1 = mid;
        }
        for (long long q = q0; q < n_right; ++q) {
            const unsigned long long rk = __ldg(rkey + q);
            const long long y = (long long)(rk >> 14);
            if (y > yhi) break;
            const int j = (int)((rk >> 4) & (PROD_MAX_PRIMERS - 1)), rm = (int)(rk & 15);
            const int lj = __ldg(plen + j);
            const long long length = y + lj - g;
            if (y < g + li || length < lo || length > hi || y + lj > end) continue;
            atomicAdd(cnt + j, 1ull);
            atomicMin(best + j, pack_best(lm + rm, length, g - o, lm));
        }
    }
    __syncthreads();
    const unsigned long long run = (unsigned long long)lrec[a] << 20 | (lkey[a] >> 47) << 10;
    for (int j = threadIdx.x; j < n_primer; j += blockDim.x) {
        if (!cnt[j]) continue;
        const unsigned long long slot = atomicAdd(n_part, 1ull);
        if ((long long)slot < cap) {
            pkey[slot] = run | (unsigned long long)j;
            pacc[slot] = ProdAcc{cnt[j], best[j]};
        }
    }
}

__global__ void k_products_summary(const unsigned long long* __restrict__ gkey, const ProdAcc* __restrict__ gacc,
                                   long long n, const uint8_t* __restrict__ list, int n_primer,
                                   unsigned long long* __restrict__ comb, uint32_t* __restrict__ recflag,
                                   uint32_t* __restrict__ listed) {
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const unsigned long long key = gkey[k];
        const long long c = (long long)((key >> 10) & (PROD_MAX_PRIMERS - 1)) * n_primer + (long long)(key & (PROD_MAX_PRIMERS - 1));
        const ProdAcc acc = gacc[k];
        const bool perfect = (acc.best >> 59) == 0;
        atomicAdd(comb + 3 * c, acc.cnt);
        atomicAdd(comb + 3 * c + 1, 1ull);
        if (perfect) atomicAdd(comb + 3 * c + 2, 1ull);
        const bool l = __ldg(list + c) != 0;
        listed[k] = l;
        if (l) atomicOr(recflag + (key >> 20), perfect ? 3u : 1u);
    }
}

// listed group -> rows[pos] = (record, i, j, start, length, left mismatches, right mismatches, products)
__global__ void k_products_rows(const unsigned long long* __restrict__ gkey, const ProdAcc* __restrict__ gacc,
                                const uint32_t* __restrict__ listed, const uint32_t* __restrict__ pos, long long n,
                                long long max_rows, int64_t* __restrict__ rows, const uint32_t* __restrict__ recflag,
                                long long n_rec, unsigned long long* __restrict__ uni) {
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        if (!listed[k] || pos[k] >= max_rows) continue;
        const unsigned long long key = gkey[k];
        const ProdAcc acc = gacc[k];
        const int tot = (int)(acc.best >> 59), lm = (int)(acc.best & 15);
        int64_t* row = rows + 8 * (long long)pos[k];
        row[0] = (int64_t)(key >> 20);
        row[1] = (int64_t)((key >> 10) & (PROD_MAX_PRIMERS - 1));
        row[2] = (int64_t)(key & (PROD_MAX_PRIMERS - 1));
        row[3] = (int64_t)((acc.best >> 4) & 0xFFFFFFFFull);
        row[4] = (int64_t)((acc.best >> 36) & ((1ull << 23) - 1));
        row[5] = lm;
        row[6] = tot - lm;
        row[7] = (int64_t)acc.cnt;
    }
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_rec; r += (long long)gridDim.x * blockDim.x) {
        const uint32_t f = recflag[r];
        if (f & 1) atomicAdd(uni, 1ull);
        if (f & 2) atomicAdd(uni + 1, 1ull);
    }
}


namespace {

// device memory owned by one call
struct DMem {
    void* p = nullptr;
    size_t bytes = 0;
    ~DMem() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
    cudaError_t reserve(size_t n) {  // contents are not kept
        if (n <= bytes) return cudaSuccess;
        release();
        cudaError_t e = cudaMalloc(&p, n);
        if (e == cudaSuccess) bytes = n;
        return e;
    }
    cudaError_t grow(size_t n, size_t keep, cudaStream_t st) {  // the first `keep` bytes are kept
        if (n <= bytes) return cudaSuccess;
        void* q = nullptr;
        cudaError_t e = cudaMalloc(&q, n);
        if (e == cudaSuccess && keep) e = cudaMemcpyAsync(q, p, keep, cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            if (q) cudaFree(q);
            return e;
        }
        release();
        p = q;
        bytes = n;
        return cudaSuccess;
    }
    template <class T>
    T* as() const {
        return (T*)p;
    }
};

// one CUB algorithm: size query, temporary storage, the run bracketed by profiling events under `name`
template <class F>
int cub_run(mpb_ctx* ctx, const char* name, DMem& tmp, F&& f) {
    size_t bytes = 0;
    CK(f((void*)nullptr, bytes));
    CK(tmp.reserve(bytes ? bytes : 1));
    ProfRec pr = {name, nullptr, nullptr, 0};
    if (ctx->profile) {
        CK(cudaEventCreate(&pr.e0));
        CK(cudaEventCreate(&pr.e1));
        CK(cudaEventRecord(pr.e0, ctx->stream));
    }
    CK(f(tmp.p, bytes));
    ctx->launches++;
    if (ctx->profile) {
        CK(cudaEventRecord(pr.e1, ctx->stream));
        ctx->recs.push_back(pr);
    }
    return 0;
}

unsigned grid_of(long long n) {
    const long long b = (n + 255) / 256;
    return (unsigned)(b < 1 ? 1 : b > 65536 ? 65536 : b);
}

int bits_for(long long n) {  // bits of the values 0..n-1
    int b = 1;
    while ((1ll << b) < n) ++b;
    return b;
}

// sort (key, acc) pairs of n groups by key and merge equal keys: in -> out, returns the merged count through *n_out
int merge_groups(mpb_ctx* ctx, DMem& tmp, DMem& d_n, int key_bits, unsigned long long* k_in, ProdAcc* v_in,
                 unsigned long long* k_tmp, ProdAcc* v_tmp, unsigned long long* k_out, ProdAcc* v_out, long long n,
                 long long* n_out) {
    int rc = cub_run(ctx, "k_products_reduce", tmp, [&](void* t, size_t& bytes) {
        return cub::DeviceRadixSort::SortPairs(t, bytes, k_in, k_tmp, v_in, v_tmp, n, 0, key_bits, ctx->stream);
    });
    if (rc) return rc;
    long long* nr = d_n.as<long long>();
    rc = cub_run(ctx, "k_products_reduce", tmp, [&](void* t, size_t& bytes) {
        return cub::DeviceReduce::ReduceByKey(t, bytes, k_tmp, k_out, v_tmp, v_out, nr, ProdMerge(), n, ctx->stream);
    });
    if (rc) return rc;
    CK(cudaMemcpyAsync(n_out, nr, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

}  // namespace

extern "C" int mpb_pattern_products(mpb_msa* m, int32_t n_pat, const uint32_t* allow, const int32_t* lens,
                                    const uint32_t* strict, int32_t v, const int32_t* pat_primer, const int32_t* pat_side,
                                    int32_t n_primer, int64_t stride, int32_t n_rec, const int64_t* rec_off,
                                    const int64_t* rec_len, int32_t lo, int32_t hi, const uint8_t* list, int64_t chunk,
                                    int64_t max_rows, int64_t* comb, int64_t* uni, int64_t* rows, int64_t* n_listed,
                                    int64_t* stats) {
    if (!m || !allow || !lens || !strict || !pat_primer || !pat_side || !list || !comb || !uni || !n_listed || !stats ||
        (n_rec > 0 && (!rec_off || !rec_len)) || (max_rows > 0 && !rows))
        return fail(MPB_EINVAL, "NULL argument");
    if (v < 0) return fail(MPB_EINVAL, "negative mismatch bound %d", v);
    if (n_pat < 1 || n_rec < 0 || max_rows < 0 || chunk < 0) return fail(MPB_EINVAL, "bad n_pat, n_rec, max_rows or chunk");
    if (n_primer < 1 || n_primer > PROD_MAX_PRIMERS)
        return fail(MPB_EINVAL, "%d primers: at most %d primers are supported", n_primer, PROD_MAX_PRIMERS);
    if (lo < 1 || lo > hi || hi > PROD_MAX_HI)
        return fail(MPB_EINVAL, "product lengths %d..%d: need 0 < lo <= hi <= %d", lo, hi, PROD_MAX_HI);
    if (stride < 1 || m->n_seq * stride >= (1ll << PROD_POS_BITS))
        return fail(MPB_EINVAL, "%lld rows of stride %lld: the stream must be shorter than 2^%d columns",
                    (long long)m->n_seq, (long long)stride, PROD_POS_BITS);
    std::vector<int32_t> plen(n_primer, 0);
    for (int p = 0; p < n_pat; ++p) {
        const int i = pat_primer[p];
        if (i < 0 || i >= n_primer || (pat_side[p] != 0 && pat_side[p] != 1))
            return fail(MPB_EINVAL, "pattern %d: primer %d / side %d out of range", p, i, pat_side[p]);
        if (plen[i] && plen[i] != lens[p])
            return fail(MPB_EINVAL, "pattern %d: length %d differs from primer %d's %d", p, lens[p], i, plen[i]);
        plen[i] = lens[p];
    }
    int lmin = 1 << 30, lmax = 0;
    for (int i = 0; i < n_primer; ++i)
        if (plen[i]) lmin = plen[i] < lmin ? plen[i] : lmin, lmax = plen[i] > lmax ? plen[i] : lmax;
    for (int r = 0; r < n_rec; ++r) {
        if (rec_len[r] < 0 || rec_len[r] > PROD_MAX_RECORD)
            return fail(MPB_EINVAL, "record %d: length %lld outside 0..%lld (the packed product start)", r,
                        (long long)rec_len[r], (long long)PROD_MAX_RECORD);
        if (rec_off[r] < 0 || (r > 0 && rec_off[r] < rec_off[r - 1] + rec_len[r - 1]))
            return fail(MPB_EINVAL, "record %d: offset %lld overlaps the record before it", r, (long long)rec_off[r]);
    }
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    const size_t ncomb = (size_t)n_primer * n_primer;
    memset(comb, 0, ncomb * 3 * sizeof(int64_t));
    uni[0] = uni[1] = 0;
    *n_listed = 0;
    for (int s = 0; s < 4; ++s) stats[s] = 0;
    if (n_rec == 0) return 0;

    // search into device buffers
    DMem hp, hr, hx, hm;
    int64_t cap = 1 << 24, n_hits = 0;  // 256 MB: one search for panels of tens of millions of sites
    for (;;) {
        CK(hp.reserve(cap * 4));
        CK(hr.reserve(cap * 4));
        CK(hx.reserve(cap * 4));
        CK(hm.reserve(cap * 4));
        const int rc = mpb_pattern_search(m, n_pat, allow, lens, strict, v, cap, hp.as<int32_t>(), hr.as<int32_t>(),
                                          hx.as<int32_t>(), hm.as<int32_t>(), &n_hits);
        if (rc) return rc;
        if (n_hits <= cap) break;
        cap = n_hits + 16;
    }
    stats[0] = n_hits;

    // filter into left / right keys
    DMem d_pp, d_ps, d_pl, d_plen, d_off, d_len, d_list, d_cnt, lk, rk, lk2, rk2, tmp;
    std::vector<int32_t> pat_len(lens, lens + n_pat);
    CK(d_pp.reserve(n_pat * 4));
    CK(d_ps.reserve(n_pat * 4));
    CK(d_pl.reserve(n_pat * 4));
    CK(d_plen.reserve(n_primer * 4));
    CK(d_off.reserve(n_rec * 8));
    CK(d_len.reserve(n_rec * 8));
    CK(d_list.reserve(ncomb));
    CK(d_cnt.reserve(64));
    CK(cudaMemcpyAsync(d_pp.p, pat_primer, n_pat * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_ps.p, pat_side, n_pat * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_pl.p, pat_len.data(), n_pat * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_plen.p, plen.data(), n_primer * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_off.p, rec_off, n_rec * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_len.p, rec_len, n_rec * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_list.p, list, ncomb, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(d_cnt.p, 0, 64, ctx->stream));
    unsigned long long* cnt = d_cnt.as<unsigned long long>();  // [0] left sites, [1] right sites, [2] partials, [3..4] union
    const long long nh = n_hits > 0 ? n_hits : 1;
    CK(lk.reserve(nh * 8));
    CK(rk.reserve(nh * 8));
    CK(lk2.reserve(nh * 8));
    CK(rk2.reserve(nh * 8));
    if (n_hits > 0)
        MPB_LAUNCH_NAMED(ctx, "k_products_filter", k_products_filter, grid_of(n_hits), 256, 0, hp.as<int32_t>(),
                         hr.as<int32_t>(), hx.as<int32_t>(), hm.as<int32_t>(), (long long)n_hits, d_pp.as<int32_t>(),
                         d_ps.as<int32_t>(), d_pl.as<int32_t>(), (long long)stride, d_off.as<int64_t>(),
                         d_len.as<int64_t>(), (int)n_rec, lk.as<unsigned long long>(), rk.as<unsigned long long>(), cnt);
    unsigned long long nlr[2];
    CK(cudaMemcpyAsync(nlr, cnt, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const long long n_left = (long long)nlr[0], n_right = (long long)nlr[1];
    stats[1] = n_left;
    stats[2] = n_right;
    hp.release(), hr.release(), hx.release(), hm.release();
    if (n_left == 0 || n_right == 0) return 0;
    if (n_left >= (1ll << 31)) return fail(MPB_EINVAL, "%lld left sites: at most 2^31 - 1 are supported", n_left);

    // sort: left sites in runs of one (primer, record), right sites in stream order
    const int pos_bits = bits_for(m->n_seq * stride);
    {
        unsigned long long *a = lk.as<unsigned long long>(), *b = lk2.as<unsigned long long>();
        int rc = cub_run(ctx, "k_products_sort", tmp, [&](void* t, size_t& bytes) {
            return cub::DeviceRadixSort::SortKeys(t, bytes, a, b, n_left, 0, 47 + bits_for(n_primer), ctx->stream);
        });
        if (rc) return rc;
        unsigned long long *c = rk.as<unsigned long long>(), *d = rk2.as<unsigned long long>();
        rc = cub_run(ctx, "k_products_sort", tmp, [&](void* t, size_t& bytes) {
            return cub::DeviceRadixSort::SortKeys(t, bytes, c, d, n_right, 0, 14 + pos_bits, ctx->stream);
        });
        if (rc) return rc;
    }
    lk.release(), rk.release();
    const unsigned long long* lkey = lk2.as<unsigned long long>();
    const unsigned long long* rkey = rk2.as<unsigned long long>();

    // segments of at most seg_len left sites inside one run; a chunk is per_chunk consecutive segments
    const long long budget = chunk > 0 ? chunk : PROD_CHUNK;
    const int seg_len = (int)(budget < PROD_SEG ? budget : PROD_SEG);
    const long long per_chunk = budget / seg_len;
    DMem d_lrec, d_head, d_hpos, d_seg;
    CK(d_lrec.reserve(n_left * 4));
    CK(d_head.reserve(n_left * 4));
    CK(d_hpos.reserve(n_left * 4));
    CK(d_seg.reserve((n_left + 1) * 4));
    MPB_LAUNCH_NAMED(ctx, "k_products_segments", k_products_heads, grid_of(n_left), 256, 0, lkey, n_left,
                     d_off.as<int64_t>(), (int)n_rec, seg_len, d_lrec.as<int32_t>(), d_head.as<uint32_t>());
    {
        const uint32_t* a = d_head.as<uint32_t>();
        uint32_t* b = d_hpos.as<uint32_t>();
        int rc = cub_run(ctx, "k_products_segments", tmp, [&](void* t, size_t& bytes) {
            return cub::DeviceScan::ExclusiveSum(t, bytes, a, b, n_left, ctx->stream);
        });
        if (rc) return rc;
    }
    MPB_LAUNCH_NAMED(ctx, "k_products_segments", k_products_segments, grid_of(n_left), 256, 0, d_head.as<uint32_t>(),
                     d_hpos.as<uint32_t>(), n_left, d_seg.as<int32_t>());
    uint32_t last[2];
    CK(cudaMemcpyAsync(last, d_hpos.as<uint32_t>() + n_left - 1, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(last + 1, d_head.as<uint32_t>() + n_left - 1, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const long long n_seg = (long long)last[0] + last[1];
    d_head.release(), d_hpos.release();

    // join chunk by chunk; a chunk's partial groups are merged before they join the groups of the earlier chunks
    DMem pk, pa, pk2, pa2, gk, ga, d_nr;
    CK(d_nr.reserve(8));
    const int key_bits = 20 + bits_for(n_rec);
    long long pcap = 1 << 20, n_groups = 0, gcap = 0;
    const size_t smem = (size_t)n_primer * 16;
    for (long long s0 = 0; s0 < n_seg; s0 += per_chunk) {
        const long long ns = n_seg - s0 < per_chunk ? n_seg - s0 : per_chunk;
        unsigned long long n_part = 0;
        for (;;) {
            CK(pk.reserve(pcap * 8));
            CK(pa.reserve(pcap * 16));
            CK(cudaMemsetAsync(cnt + 2, 0, 8, ctx->stream));
            MPB_LAUNCH_NAMED(ctx, "k_products_join", k_products_join, (unsigned)ns, PROD_SEG, smem, lkey,
                             d_lrec.as<int32_t>(), d_seg.as<int32_t>(), s0, rkey, n_right, d_plen.as<int32_t>(),
                             (int)n_primer, lmin, lmax, (int)lo, (int)hi, d_off.as<int64_t>(), d_len.as<int64_t>(),
                             pk.as<unsigned long long>(), pa.as<ProdAcc>(), cnt + 2, pcap);
            CK(cudaMemcpyAsync(&n_part, cnt + 2, 8, cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            if ((long long)n_part <= pcap) break;
            pcap = (long long)n_part + 16;
        }
        if (n_part == 0) continue;
        const long long np = (long long)n_part;
        if (n_groups + np > gcap) {
            const long long want = n_groups + np > 2 * gcap ? n_groups + np : 2 * gcap;
            CK(gk.grow(want * 8, n_groups * 8, ctx->stream));
            CK(ga.grow(want * 16, n_groups * 16, ctx->stream));
            gcap = want;
        }
        CK(pk2.reserve(np * 8));
        CK(pa2.reserve(np * 16));
        long long nr = 0;
        int rc = merge_groups(ctx, tmp, d_nr, key_bits, pk.as<unsigned long long>(), pa.as<ProdAcc>(),
                              pk2.as<unsigned long long>(), pa2.as<ProdAcc>(), gk.as<unsigned long long>() + n_groups,
                              ga.as<ProdAcc>() + n_groups, np, &nr);
        if (rc) return rc;
        n_groups += nr;
    }
    pk.release(), pa.release(), pk2.release(), pa2.release(), d_lrec.release(), d_seg.release(), lk2.release(), rk2.release();
    if (n_groups == 0) return 0;
    if (n_seg > per_chunk) {  // a run cut by a chunk boundary left one partial group on each side
        DMem k2, a2;
        CK(k2.reserve(n_groups * 8));
        CK(a2.reserve(n_groups * 16));
        long long nr = 0;
        int rc = merge_groups(ctx, tmp, d_nr, key_bits, gk.as<unsigned long long>(), ga.as<ProdAcc>(),
                              k2.as<unsigned long long>(), a2.as<ProdAcc>(), gk.as<unsigned long long>(),
                              ga.as<ProdAcc>(), n_groups, &nr);
        if (rc) return rc;
        n_groups = nr;
    }
    stats[3] = n_groups;
    if (n_groups >= (1ll << 32)) return fail(MPB_EINVAL, "%lld groups: at most 2^32 - 1 are supported", n_groups);

    // summary, listed rows, union
    DMem d_comb, d_flag, d_listed, d_lpos, d_rows;
    const long long n_out = max_rows < n_groups ? max_rows : n_groups;
    CK(d_comb.reserve(ncomb * 3 * 8));
    CK(d_flag.reserve((size_t)n_rec * 4));
    CK(d_listed.reserve(n_groups * 4));
    CK(d_lpos.reserve(n_groups * 4));
    CK(d_rows.reserve((n_out > 0 ? n_out : 1) * 64));
    CK(cudaMemsetAsync(d_comb.p, 0, ncomb * 3 * 8, ctx->stream));
    CK(cudaMemsetAsync(d_flag.p, 0, (size_t)n_rec * 4, ctx->stream));
    MPB_LAUNCH_NAMED(ctx, "k_products_summary", k_products_summary, grid_of(n_groups), 256, 0, gk.as<unsigned long long>(),
                     ga.as<ProdAcc>(), n_groups, d_list.as<uint8_t>(), (int)n_primer, d_comb.as<unsigned long long>(),
                     d_flag.as<uint32_t>(), d_listed.as<uint32_t>());
    {
        const uint32_t* a = d_listed.as<uint32_t>();
        uint32_t* b = d_lpos.as<uint32_t>();
        int rc = cub_run(ctx, "k_products_summary", tmp, [&](void* t, size_t& bytes) {
            return cub::DeviceScan::ExclusiveSum(t, bytes, a, b, n_groups, ctx->stream);
        });
        if (rc) return rc;
    }
    MPB_LAUNCH_NAMED(ctx, "k_products_summary", k_products_rows, grid_of(n_groups > n_rec ? n_groups : n_rec), 256, 0,
                     gk.as<unsigned long long>(), ga.as<ProdAcc>(), d_listed.as<uint32_t>(), d_lpos.as<uint32_t>(),
                     n_groups, (long long)n_out, d_rows.as<int64_t>(), d_flag.as<uint32_t>(), (long long)n_rec, cnt + 3);
    uint32_t lastl[2];
    unsigned long long u[2];
    CK(cudaMemcpyAsync(comb, d_comb.p, ncomb * 3 * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(u, cnt + 3, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(lastl, d_lpos.as<uint32_t>() + n_groups - 1, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(lastl + 1, d_listed.as<uint32_t>() + n_groups - 1, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *n_listed = (int64_t)lastl[0] + lastl[1];
    const long long n_copy = *n_listed < n_out ? *n_listed : n_out;
    if (n_copy > 0) CK(cudaMemcpyAsync(rows, d_rows.p, n_copy * 64, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    uni[0] = (int64_t)u[0];
    uni[1] = (int64_t)u[1];
    return 0;
}


// ---- mpb_pattern_cover / mpb_cover_gains / mpb_cover_take (primer_select.py) ---------------------------------------
// Each pair's own amplicons only, as one bit per (pair, record) that stays in HBM:
//   search   k_pattern_sites into device buffers, as above;
//   filter   k_cover_filter: the sites k_products_filter keeps, each packed into one 64-bit key
//              pattern << (pos_bits + 4) | stream position << 4 | mismatches
//            so one sort puts every pattern's sites in stream order, the runs of 4q .. 4q+3 one after the other;
//   sort     cub::DeviceRadixSort of the keys;
//   join     k_cover_join: a thread per left site (pattern 4q: F, 4q+2: R) binary-searches the run of its right pattern
//            (4q+1: RC(R), 4q+3: RC(F)) for the first site in the product window; any site there is an amplicon, so it
//            sets the record's bit of pair q, and the perfect bit when the left site and some right site in the window
//            have no mismatch.  Only sites and bits are stored, never products.
#define COVER_MAX_REC ((1ll << 31) - 1)

__global__ void k_cover_filter(const int32_t* __restrict__ hp, const int32_t* __restrict__ hr, const int32_t* __restrict__ hx,
                               const int32_t* __restrict__ hm, long long n, const int32_t* __restrict__ pat_len,
                               long long stride, const int64_t* __restrict__ off, const int64_t* __restrict__ len,
                               int n_rec, int pos_bits, unsigned long long* __restrict__ key,
                               unsigned long long* __restrict__ n_key) {
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const long long x = hx[k];
        if (x >= stride) continue;
        const long long g = (long long)hr[k] * stride + x;
        const int r = find_record(off, n_rec, g);
        if (r < 0) continue;
        const int p = hp[k];
        if (g + __ldg(pat_len + p) > __ldg(off + r) + __ldg(len + r)) continue;
        const unsigned long long slot = atomicAdd(n_key, 1ull);
        key[slot] = (unsigned long long)p << (pos_bits + 4) | (unsigned long long)g << 4 | (unsigned long long)hm[k];
        if ((p & 1) == 0) atomicAdd(n_key + 1, 1ull);  // left sites
    }
}

__global__ void k_cover_join(const unsigned long long* __restrict__ key, long long n, int pos_bits,
                             const int32_t* __restrict__ pat_len, int lo, int hi, const int64_t* __restrict__ off,
                             const int64_t* __restrict__ len, int n_rec, long long words, uint32_t* __restrict__ amp,
                             uint32_t* __restrict__ perf) {
    const unsigned long long pos_mask = (1ull << pos_bits) - 1;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const unsigned long long kk = key[k];
        const int p = (int)(kk >> (pos_bits + 4));
        if (p & 1) continue;  // right sites are what the left sites look for
        const long long g = (long long)((kk >> 4) & pos_mask);
        const int lm = (int)(kk & 15);
        const int r = find_record(off, n_rec, g);
        const long long end = __ldg(off + r) + __ldg(len + r);
        const int ll = __ldg(pat_len + p), rl = __ldg(pat_len + p + 1);
        const long long ylo = g + max(ll, lo - rl), yhi = min(g + (long long)hi - rl, end - rl);
        if (ylo > yhi) continue;
        const unsigned long long base = (unsigned long long)(p + 1) << (pos_bits + 4);
        const unsigned long long want = base | (unsigned long long)ylo << 4, last = base | (unsigned long long)yhi << 4 | 15;
        long long q0 = k + 1, q1 = n;  // the right run follows the left one
        while (q0 < q1) {
            const long long mid = (q0 + q1) >> 1;
            if (__ldg(key + mid) < want) q0 = mid + 1;
            else q1 = mid;
        }
        if (q0 >= n || __ldg(key + q0) > last) continue;
        const long long word = (long long)(p >> 2) * words + (r >> 5);
        const uint32_t bit = 1u << (r & 31);
        if (!(__ldcg(amp + word) & bit)) atomicOr(amp + word, bit);
        if (lm != 0 || (__ldcg(perf + word) & bit)) continue;
        for (long long q = q0; q < n; ++q) {  // stop at the first perfect product
            const unsigned long long rk = __ldg(key + q);
            if (rk > last) break;
            if ((rk & 15) == 0) {
                atomicOr(perf + word, bit);
                break;
            }
        }
    }
}

// the site list of mpb_pattern_cover_keep (defined below)
static int sites_check_block(const mpb_site_list* s, int32_t pat0, int32_t n_pat, const int32_t* lens, int32_t n_rec,
                             const int64_t* rec_off, const int64_t* rec_len);
static int sites_append(mpb_site_list* s, const unsigned long long* key, long long n, int pos_bits, int32_t pat0);

// mpb_pattern_cover, and with a site list (list != NULL) mpb_pattern_cover_keep: the same search, filter, sort and join,
// with the filtered sites also appended to the list; amp / perf NULL (keep only) stops after the append
static int pattern_cover(mpb_msa* m, int32_t n_pat, const uint32_t* allow, const int32_t* lens, const uint32_t* strict,
                         int32_t v, int64_t stride, int32_t n_rec, const int64_t* rec_off, const int64_t* rec_len,
                         int32_t lo, int32_t hi, int64_t words, uint32_t* amp, uint32_t* perf, int64_t max_sites,
                         int64_t* stats, mpb_site_list* list, int32_t pat0) {
    const bool join = amp || perf || !list;
    if (!m || !allow || !lens || !strict || (join && (!amp || !perf)) || !stats || (n_rec > 0 && (!rec_off || !rec_len)))
        return fail(MPB_EINVAL, "NULL argument");
    if (v < 0) return fail(MPB_EINVAL, "negative mismatch bound %d", v);
    if (n_pat < 4 || n_pat % 4) return fail(MPB_EINVAL, "%d patterns: four per pair are needed", n_pat);
    if (n_rec < 0 || (long long)n_rec > COVER_MAX_REC) return fail(MPB_EINVAL, "bad n_rec %d", n_rec);
    if (join && words < (n_rec + 31) / 32)
        return fail(MPB_EINVAL, "%lld words hold fewer than %d records", (long long)words, n_rec);
    if (lo < 1 || lo > hi) return fail(MPB_EINVAL, "product lengths %d..%d: need 0 < lo <= hi", lo, hi);
    if (max_sites < 0 || max_sites > (1ll << 31)) return fail(MPB_EINVAL, "max_sites %lld outside 0..2^31", (long long)max_sites);
    if (join && (!mpb_is_device_ptr(amp) || !mpb_is_device_ptr(perf)))
        return fail(MPB_EINVAL, "amp and perf must be device memory");
    if (stride < 1 || stride > (1ll << 60) / (m->n_seq > 0 ? m->n_seq : 1))
        return fail(MPB_EINVAL, "%lld rows of stride %lld: the site key needs more than 64 bits", (long long)m->n_seq,
                    (long long)stride);
    const int pat_bits = bits_for(n_pat), pos_bits = bits_for(m->n_seq * stride);
    if (pat_bits + pos_bits + 4 > 64)
        return fail(MPB_EINVAL, "%d patterns over %lld rows of stride %lld: the site key needs %d + %d + 4 > 64 bits", n_pat,
                    (long long)m->n_seq, (long long)stride, pat_bits, pos_bits);
    for (int r = 0; r < n_rec; ++r)
        if (rec_len[r] < 0 || rec_off[r] < 0 || (r > 0 && rec_off[r] < rec_off[r - 1] + rec_len[r - 1]))
            return fail(MPB_EINVAL, "record %d: offset %lld / length %lld overlap the record before it", r,
                        (long long)rec_off[r], (long long)rec_len[r]);
    if (n_rec > 0 && rec_off[n_rec - 1] + rec_len[n_rec - 1] > m->n_seq * stride)  // keys and windows stay in pos_bits
        return fail(MPB_EINVAL, "record %d ends at %lld, past the %lld stream columns of the rows", n_rec - 1,
                    (long long)(rec_off[n_rec - 1] + rec_len[n_rec - 1]), (long long)(m->n_seq * stride));
    if (list)
        if (int rc = sites_check_block(list, pat0, n_pat, lens, n_rec, rec_off, rec_len)) return rc;
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    for (int s = 0; s < 3; ++s) stats[s] = 0;
    if (n_rec == 0) return 0;

    // the search runs once when the caller's capacity holds its sites, twice otherwise (counted, then stored)
    DMem hp, hr, hx, hm;
    int64_t cap = max_sites > 0 ? max_sites : 1 << 24, n_hits = 0;
    for (;;) {
        CK(hp.reserve(cap * 4));
        CK(hr.reserve(cap * 4));
        CK(hx.reserve(cap * 4));
        CK(hm.reserve(cap * 4));
        const int rc = mpb_pattern_search(m, n_pat, allow, lens, strict, v, cap, hp.as<int32_t>(), hr.as<int32_t>(),
                                          hx.as<int32_t>(), hm.as<int32_t>(), &n_hits);
        if (rc) return rc;
        if (n_hits <= cap) break;
        cap = n_hits + 16;
    }
    stats[0] = n_hits;

    DMem d_pl, d_off, d_len, d_cnt, k1, k2, tmp;
    CK(d_pl.reserve(n_pat * 4));
    CK(d_off.reserve(n_rec * 8));
    CK(d_len.reserve(n_rec * 8));
    CK(d_cnt.reserve(16));
    CK(cudaMemcpyAsync(d_pl.p, lens, n_pat * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_off.p, rec_off, n_rec * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_len.p, rec_len, n_rec * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(d_cnt.p, 0, 16, ctx->stream));
    const long long nh = n_hits > 0 ? n_hits : 1;
    CK(k1.reserve(nh * 8));
    CK(k2.reserve(nh * 8));
    unsigned long long* cnt = d_cnt.as<unsigned long long>();
    if (n_hits > 0)
        MPB_LAUNCH_NAMED(ctx, "k_cover_filter", k_cover_filter, grid_of(n_hits), 256, 0, hp.as<int32_t>(), hr.as<int32_t>(),
                         hx.as<int32_t>(), hm.as<int32_t>(), (long long)n_hits, d_pl.as<int32_t>(), (long long)stride,
                         d_off.as<int64_t>(), d_len.as<int64_t>(), (int)n_rec, pos_bits, k1.as<unsigned long long>(), cnt);
    unsigned long long nk[2];
    CK(cudaMemcpyAsync(nk, cnt, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    hp.release(), hr.release(), hx.release(), hm.release();
    const long long n_key = (long long)nk[0];
    stats[1] = (int64_t)nk[1];
    stats[2] = n_key - (int64_t)nk[1];
    if (list)
        if (int rc = sites_append(list, k1.as<unsigned long long>(), n_key, pos_bits, pat0)) return rc;
    if (!join || stats[1] == 0 || stats[2] == 0) return 0;
    {
        unsigned long long *a = k1.as<unsigned long long>(), *b = k2.as<unsigned long long>();
        const int rc = cub_run(ctx, "k_cover_sort", tmp, [&](void* t, size_t& bytes) {
            return cub::DeviceRadixSort::SortKeys(t, bytes, a, b, n_key, 0, pat_bits + pos_bits + 4, ctx->stream);
        });
        if (rc) return rc;
    }
    k1.release();
    MPB_LAUNCH_NAMED(ctx, "k_cover_join", k_cover_join, grid_of(n_key), 256, 0, k2.as<unsigned long long>(), n_key,
                     pos_bits, d_pl.as<int32_t>(), (int)lo, (int)hi, d_off.as<int64_t>(), d_len.as<int64_t>(), (int)n_rec,
                     (long long)words, amp, perf);
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int mpb_pattern_cover(mpb_msa* m, int32_t n_pat, const uint32_t* allow, const int32_t* lens,
                                 const uint32_t* strict, int32_t v, int64_t stride, int32_t n_rec, const int64_t* rec_off,
                                 const int64_t* rec_len, int32_t lo, int32_t hi, int64_t words, uint32_t* amp,
                                 uint32_t* perf, int64_t max_sites, int64_t* stats) {
    return pattern_cover(m, n_pat, allow, lens, strict, v, stride, n_rec, rec_off, rec_len, lo, hi, words, amp, perf,
                         max_sites, stats, nullptr, 0);
}

extern "C" int mpb_pattern_cover_keep(mpb_msa* m, int32_t n_pat, const uint32_t* allow, const int32_t* lens,
                                      const uint32_t* strict, int32_t v, int64_t stride, int32_t n_rec,
                                      const int64_t* rec_off, const int64_t* rec_len, int32_t lo, int32_t hi, int64_t words,
                                      uint32_t* amp, uint32_t* perf, int64_t max_sites, int64_t* stats,
                                      mpb_site_list* list, int32_t pat0) {
    if (!list) return fail(MPB_EINVAL, "NULL site list");
    if ((amp == nullptr) != (perf == nullptr)) return fail(MPB_EINVAL, "amp and perf: both or neither");
    return pattern_cover(m, n_pat, allow, lens, strict, v, stride, n_rec, rec_off, rec_len, lo, hi, words, amp, perf,
                         max_sites, stats, list, pat0);
}

// gains[2i] = popcount(amp[cand[i]] & ~covered), gains[2i+1] = popcount(perf[cand[i]] & ~covered_perfect): one warp per
// listed row, 128-bit loads, a warp-shuffle sum and one store per row; rows that are not listed are never read
#define GAINS_WARPS 8
__global__ void __launch_bounds__(GAINS_WARPS * 32)
k_cover_gains(const uint4* __restrict__ amp, const uint4* __restrict__ perf, long long words4,
              const uint4* __restrict__ cov, const uint4* __restrict__ covp, const int32_t* __restrict__ cand, long long n,
              int64_t* __restrict__ gains) {
    const long long i = (long long)blockIdx.x * GAINS_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const long long row = (long long)__ldg(cand + i) * words4;
    unsigned a = 0, b = 0;
    for (long long w = lane; w < words4; w += 32) {
        const uint4 x = __ldg(amp + row + w), y = __ldg(perf + row + w), c = __ldg(cov + w), d = __ldg(covp + w);
        a += __popc(x.x & ~c.x) + __popc(x.y & ~c.y) + __popc(x.z & ~c.z) + __popc(x.w & ~c.w);
        b += __popc(y.x & ~d.x) + __popc(y.y & ~d.y) + __popc(y.z & ~d.z) + __popc(y.w & ~d.w);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        a += __shfl_xor_sync(0xFFFFFFFFu, a, s);
        b += __shfl_xor_sync(0xFFFFFFFFu, b, s);
    }
    if (lane == 0) {
        gains[2 * i] = a;
        gains[2 * i + 1] = b;
    }
}

__global__ void k_cover_take(const uint32_t* __restrict__ amp, const uint32_t* __restrict__ perf, long long words,
                             uint32_t* __restrict__ cov, uint32_t* __restrict__ covp) {
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < words; w += (long long)gridDim.x * blockDim.x) {
        cov[w] |= amp[w];
        covp[w] |= perf[w];
    }
}

static int cover_args(const uint32_t* amp, const uint32_t* perf, int64_t n_rows, int64_t words, const uint32_t* cov,
                      const uint32_t* covp) {
    if (!amp || !perf || !cov || !covp) return fail(MPB_EINVAL, "NULL argument");
    if (n_rows < 0 || words < 4 || words % 4)
        return fail(MPB_EINVAL, "%lld rows of %lld words: need rows >= 0 and words a positive multiple of 4",
                    (long long)n_rows, (long long)words);
    for (const void* p : {(const void*)amp, (const void*)perf, (const void*)cov, (const void*)covp})
        if (((uintptr_t)p & 15) || !mpb_is_device_ptr(p))
            return fail(MPB_EINVAL, "amp, perf and the covered vectors must be 16-byte aligned device memory");
    return 0;
}

extern "C" int mpb_cover_gains(mpb_ctx* ctx, const uint32_t* amp, const uint32_t* perf, int64_t n_rows, int64_t words,
                               const uint32_t* covered, const uint32_t* covered_perfect, const int32_t* cand,
                               int64_t n_cand, int64_t* gains) {
    if (!ctx || (n_cand > 0 && (!cand || !gains))) return fail(MPB_EINVAL, "NULL argument");
    if (int rc = cover_args(amp, perf, n_rows, words, covered, covered_perfect)) return rc;
    if (n_cand < 0 || n_cand > (1ll << 31) - 1) return fail(MPB_EINVAL, "bad n_cand %lld", (long long)n_cand);
    for (int64_t i = 0; i < n_cand; ++i)
        if (cand[i] < 0 || cand[i] >= n_rows)
            return fail(MPB_EINVAL, "candidate %lld: row %d outside 0..%lld", (long long)i, cand[i], (long long)n_rows - 1);
    if (n_cand == 0) return 0;
    CK(cudaSetDevice(ctx->device));
    InBuf ic(ctx, cand, (size_t)n_cand * 4);
    OutBuf og(ctx, gains, (size_t)n_cand * 16);
    if (ic.rc || og.rc) return MPB_ECUDA;
    ctx->pending_units = (double)n_cand * (double)words * 8.0;  // bytes of the listed rows
    MPB_LAUNCH(ctx, k_cover_gains, (unsigned)((n_cand + GAINS_WARPS - 1) / GAINS_WARPS), GAINS_WARPS * 32, 0,
               (const uint4*)amp, (const uint4*)perf, (long long)(words / 4), (const uint4*)covered,
               (const uint4*)covered_perfect, ic.dev<int32_t>(), (long long)n_cand, og.dev<int64_t>());
    CK(og.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int mpb_cover_take(mpb_ctx* ctx, const uint32_t* amp, const uint32_t* perf, int64_t n_rows, int64_t words,
                              int64_t row, uint32_t* covered, uint32_t* covered_perfect) {
    if (!ctx) return fail(MPB_EINVAL, "NULL argument");
    if (int rc = cover_args(amp, perf, n_rows, words, covered, covered_perfect)) return rc;
    if (row < 0 || row >= n_rows) return fail(MPB_EINVAL, "row %lld outside 0..%lld", (long long)row, (long long)n_rows - 1);
    CK(cudaSetDevice(ctx->device));
    MPB_LAUNCH(ctx, k_cover_take, grid_of(words), 256, 0, amp + row * words, perf + row * words, (long long)words, covered,
               covered_perfect);
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}


// ---- mpb_site_list: the kept sites of mpb_pattern_cover_keep and their joins (primer_select.py --cross / --background)
// The list holds the filtered sites of every pattern of a panel over one set of records, in one 64-bit key each:
//     stream position << (pat_bits + 4) | pattern << 4 | mismatches
//   keep   mpb_pattern_cover_keep appends the keys of its block (k_sites_keep re-packs the cover keys, pattern + pat0);
//   seal   one cub::DeviceRadixSort of all the keys puts them in stream order, and k_sites_count counts each pattern's
//          sites (the capacity of a pair's pick);
//   cross  k_sites_pick gathers the sites of the taken pair's four patterns, then k_sites_cross gives every one of them
//          a warp that walks the stream-ordered list from its site over its product window: forward from a left site
//          to the right sites that can close a product with it, backward from a right site to the left sites.  The
//          window is a contiguous run of the list, so the lanes read consecutive keys; a key of an eligible pair
//          (bitmask in shared memory) that closes a product sets one of its pair's 8 bits (check, then atomicOr);
//   own    k_sites_repack re-keys the list pattern-first, one sort puts each pattern's sites in stream order, and
//          k_sites_own binary-searches, for every left site, the runs of its own pair's two right patterns, as
//          k_cover_join does for one of them.
// A pattern's primer: 4q (F, left), 4q+1 (R, right), 4q+2 (R, left), 4q+3 (F, right); 0 = F, 1 = R.
struct mpb_site_list {
    mpb_ctx* ctx;
    int32_t n_pat, n_rec;
    int64_t n_pos;
    int pat_bits, pos_bits;
    std::vector<int32_t> h_lens;
    std::vector<int64_t> h_off, h_len, count;  // count: sites per pattern, after the seal
    DMem keys, d_lens, d_off, d_len;
    long long n = 0;
    bool sealed = false;
};

__device__ __forceinline__ int primer_of(int p) { return ((p & 3) == 1 || (p & 3) == 2) ? 1 : 0; }

// bit b of pair c's byte in out[] (4 pairs per word), read first so a bit that is set costs no atomic
__device__ __forceinline__ void set_pair_bit(uint32_t* out, int c, int b) {
    const uint32_t bit = 1u << ((c & 3) * 8 + b);
    if (!(__ldcg(out + (c >> 2)) & bit)) atomicOr(out + (c >> 2), bit);
}

__global__ void k_sites_keep(const unsigned long long* __restrict__ in, long long n, int in_pos_bits, int pat_bits,
                             int pat0, unsigned long long* __restrict__ out) {
    const unsigned long long pos_mask = (1ull << in_pos_bits) - 1;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const unsigned long long kk = in[k];
        const unsigned long long p = (kk >> (in_pos_bits + 4)) + (unsigned long long)pat0, g = (kk >> 4) & pos_mask;
        out[k] = g << (pat_bits + 4) | p << 4 | (kk & 15);
    }
}

__global__ void k_sites_count(const unsigned long long* __restrict__ key, long long n, int pat_bits,
                              unsigned long long* __restrict__ count) {
    const unsigned long long pat_mask = (1ull << pat_bits) - 1;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x)
        atomicAdd(count + ((key[k] >> 4) & pat_mask), 1ull);
}

__global__ void k_sites_pick(const unsigned long long* __restrict__ key, long long n, int pat_bits, int p0,
                             long long* __restrict__ pick, unsigned long long* __restrict__ n_pick) {
    const unsigned long long pat_mask = (1ull << pat_bits) - 1;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const int p = (int)((__ldg(key + k) >> 4) & pat_mask);
        if (p >= p0 && p < p0 + 4) pick[atomicAdd(n_pick, 1ull)] = k;
    }
}

#define CROSS_WARPS 8
__global__ void __launch_bounds__(CROSS_WARPS * 32)
k_sites_cross(const unsigned long long* __restrict__ key, long long n, const long long* __restrict__ pick, long long n_pick,
              int pat_bits, const int32_t* __restrict__ pat_len, const int64_t* __restrict__ off,
              const int64_t* __restrict__ len, int n_rec, int lo, int hi, const uint32_t* __restrict__ elig, int elig_words,
              uint32_t* __restrict__ out) {
    extern __shared__ uint32_t s_elig[];
    for (int w = threadIdx.x; w < elig_words; w += blockDim.x) s_elig[w] = __ldg(elig + w);
    __syncthreads();
    const long long i = (long long)blockIdx.x * CROSS_WARPS + (threadIdx.x >> 5);
    if (i >= n_pick) return;  // the whole warp
    const int lane = threadIdx.x & 31, sh = pat_bits + 4;
    const unsigned long long pat_mask = (1ull << pat_bits) - 1;
    const long long k = __ldg(pick + i);
    const unsigned long long kk = __ldg(key + k);
    const long long g = (long long)(kk >> sh);
    const int p = (int)((kk >> 4) & pat_mask), lt = __ldg(pat_len + p), pt = primer_of(p);
    const int r = find_record(off, n_rec, g);
    const long long start = __ldg(off + r), end = start + __ldg(len + r);
    if ((p & 1) == 0) {
        // a left site of the taken pair at g: right sites y >= g + lt with y + L - g in [lo, hi], y + L <= end
        const long long last = min(g + (long long)hi, end) - 1;
        for (long long b = k + 1 + lane;; b += 32) {
            bool past = b >= n;
            if (!past) {
                const unsigned long long rk = __ldg(key + b);
                const long long y = (long long)(rk >> sh);
                past = y > last;
                const int q = (int)((rk >> 4) & pat_mask), c = q >> 2;
                if (!past && (q & 1) && (s_elig[c >> 5] >> (c & 31) & 1)) {
                    const long long l = y + __ldg(pat_len + q) - g;
                    if (y >= g + lt && l >= lo && l <= hi && g + l <= end) set_pair_bit(out, c, primer_of(q) << 1 | pt);
                }
            }
            if (__any_sync(0xFFFFFFFFu, past)) break;  // the list is in stream order: every later key is past too
        }
    } else {
        // a right site of the taken pair at g: left sites x >= start with x + L <= g and g + lt - x in [lo, hi]
        const long long first = max(start, g + lt - (long long)hi);
        for (long long b = k - 1 - lane;; b -= 32) {
            bool past = b < 0;
            if (!past) {
                const unsigned long long lk = __ldg(key + b);
                const long long x = (long long)(lk >> sh);
                past = x < first;
                const int q = (int)((lk >> 4) & pat_mask), c = q >> 2;
                if (!past && !(q & 1) && (s_elig[c >> 5] >> (c & 31) & 1)) {
                    const long long l = g + lt - x;
                    if (x + __ldg(pat_len + q) <= g && l >= lo && l <= hi)
                        set_pair_bit(out, c, 4 | primer_of(q) << 1 | pt);
                }
            }
            if (__any_sync(0xFFFFFFFFu, past)) break;
        }
    }
}

__global__ void k_sites_repack(const unsigned long long* __restrict__ in, long long n, int pat_bits, int pos_bits,
                               unsigned long long* __restrict__ out) {
    const unsigned long long pat_mask = (1ull << pat_bits) - 1;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const unsigned long long kk = in[k];
        out[k] = ((kk >> 4) & pat_mask) << (pos_bits + 4) | (kk >> (pat_bits + 4)) << 4 | (kk & 15);
    }
}

__global__ void k_sites_own(const unsigned long long* __restrict__ key, long long n, int pos_bits,
                            const int32_t* __restrict__ pat_len, const int64_t* __restrict__ off,
                            const int64_t* __restrict__ len, int n_rec, int lo, int hi, uint32_t* __restrict__ out) {
    const unsigned long long pos_mask = (1ull << pos_bits) - 1;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
        const unsigned long long kk = key[k];
        const int p = (int)(kk >> (pos_bits + 4));
        if (p & 1) continue;
        const long long g = (long long)((kk >> 4) & pos_mask);
        const int r = find_record(off, n_rec, g);
        const long long end = __ldg(off + r) + __ldg(len + r);
        const int ll = __ldg(pat_len + p), c = p >> 2;
        for (int rp = (p & ~3) + 1; rp < (p & ~3) + 4; rp += 2) {  // RC(R) and RC(F) of the site's own pair
            const int b = primer_of(p) << 1 | primer_of(rp);
            if (__ldcg(out + (c >> 2)) >> ((c & 3) * 8 + b) & 1) continue;
            const int rl = __ldg(pat_len + rp);
            const long long ylo = g + max(ll, lo - rl), yhi = min(g + (long long)hi - rl, end - rl);
            if (ylo > yhi) continue;
            const unsigned long long base = (unsigned long long)rp << (pos_bits + 4);
            const unsigned long long want = base | (unsigned long long)ylo << 4, last = base | (unsigned long long)yhi << 4 | 15;
            long long q0 = 0, q1 = n;
            while (q0 < q1) {
                const long long mid = (q0 + q1) >> 1;
                if (__ldg(key + mid) < want) q0 = mid + 1;
                else q1 = mid;
            }
            if (q0 < n && __ldg(key + q0) <= last) set_pair_bit(out, c, b);
        }
    }
}

static int sites_no_memory(const char* what, long long sites, long long bytes) {
    cudaGetLastError();
    return fail(MPB_ENOMEM, "the site list's %s of %lld sites needs %lld bytes of device memory", what, sites, bytes);
}

static int sites_check_block(const mpb_site_list* s, int32_t pat0, int32_t n_pat, const int32_t* lens, int32_t n_rec,
                             const int64_t* rec_off, const int64_t* rec_len) {
    if (s->sealed) return fail(MPB_EINVAL, "the site list is sealed: no site can be added");
    if (pat0 < 0 || pat0 % 4 || (long long)pat0 + n_pat > s->n_pat)
        return fail(MPB_EINVAL, "patterns %d..%lld outside the site list's 0..%d", pat0, (long long)pat0 + n_pat - 1,
                    s->n_pat - 1);
    for (int32_t p = 0; p < n_pat; ++p)
        if (lens[p] != s->h_lens[pat0 + p])
            return fail(MPB_EINVAL, "pattern %d: length %d, the site list has %d", pat0 + p, lens[p], s->h_lens[pat0 + p]);
    if (n_rec != s->n_rec) return fail(MPB_EINVAL, "%d records, the site list has %d", n_rec, s->n_rec);
    for (int32_t r = 0; r < n_rec; ++r)
        if (rec_off[r] != s->h_off[r] || rec_len[r] != s->h_len[r])
            return fail(MPB_EINVAL, "record %d differs from the site list's", r);
    return 0;
}

static int sites_append(mpb_site_list* s, const unsigned long long* key, long long n, int pos_bits, int32_t pat0) {
    if (n == 0) return 0;
    mpb_ctx* ctx = s->ctx;
    const long long need = s->n + n;
    if ((size_t)need * 8 > s->keys.bytes) {
        const long long want = need + need / 2;  // room for the next blocks: geometric growth
        if (s->keys.grow((size_t)want * 8, (size_t)s->n * 8, ctx->stream) != cudaSuccess &&
            s->keys.grow((size_t)need * 8, (size_t)s->n * 8, ctx->stream) != cudaSuccess)
            return sites_no_memory("keys", need, need * 8);
    }
    MPB_LAUNCH(ctx, k_sites_keep, grid_of(n), 256, 0, key, n, pos_bits, s->pat_bits, (int)pat0,
               s->keys.as<unsigned long long>() + s->n);
    s->n = need;
    return 0;
}

extern "C" int mpb_site_list_create(mpb_ctx* ctx, int32_t n_pat, const int32_t* lens, int64_t n_pos, int32_t n_rec,
                                    const int64_t* rec_off, const int64_t* rec_len, mpb_site_list** out) {
    if (!ctx || !lens || !out || (n_rec > 0 && (!rec_off || !rec_len))) return fail(MPB_EINVAL, "NULL argument");
    *out = nullptr;
    if (n_pat < 4 || n_pat % 4) return fail(MPB_EINVAL, "%d patterns: four per pair are needed", n_pat);
    if (n_rec < 0 || (long long)n_rec > COVER_MAX_REC) return fail(MPB_EINVAL, "bad n_rec %d", n_rec);
    if (n_pos < 1) return fail(MPB_EINVAL, "bad n_pos %lld", (long long)n_pos);
    const int pat_bits = bits_for(n_pat), pos_bits = bits_for(n_pos);
    if (pat_bits + pos_bits + 4 > 64)
        return fail(MPB_EINVAL, "%d patterns over %lld stream columns: the site key needs %d + %d + 4 > 64 bits", n_pat,
                    (long long)n_pos, pat_bits, pos_bits);
    for (int32_t p = 0; p < n_pat; ++p)
        if (lens[p] < 1 || lens[p] > 32) return fail(MPB_EINVAL, "pattern %d: length %d outside 1..32", p, lens[p]);
    for (int32_t r = 0; r < n_rec; ++r)
        if (rec_len[r] < 0 || rec_off[r] < 0 || (r > 0 && rec_off[r] < rec_off[r - 1] + rec_len[r - 1]))
            return fail(MPB_EINVAL, "record %d: offset %lld / length %lld overlap the record before it", r,
                        (long long)rec_off[r], (long long)rec_len[r]);
    if (n_rec > 0 && rec_off[n_rec - 1] + rec_len[n_rec - 1] > n_pos)
        return fail(MPB_EINVAL, "record %d ends past the %lld stream columns", n_rec - 1, (long long)n_pos);
    CK(cudaSetDevice(ctx->device));
    mpb_site_list* s = new mpb_site_list();
    s->ctx = ctx, s->n_pat = n_pat, s->n_rec = n_rec, s->n_pos = n_pos, s->pat_bits = pat_bits, s->pos_bits = pos_bits;
    s->h_lens.assign(lens, lens + n_pat);
    s->h_off.assign(rec_off, rec_off + n_rec);
    s->h_len.assign(rec_len, rec_len + n_rec);
    cudaError_t e = s->d_lens.reserve(n_pat * 4);
    if (e == cudaSuccess) e = s->d_off.reserve(n_rec * 8 + 8);
    if (e == cudaSuccess) e = s->d_len.reserve(n_rec * 8 + 8);
    if (e == cudaSuccess) e = cudaMemcpy(s->d_lens.p, lens, n_pat * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && n_rec) e = cudaMemcpy(s->d_off.p, rec_off, n_rec * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && n_rec) e = cudaMemcpy(s->d_len.p, rec_len, n_rec * 8, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        delete s;
        CK(e);
    }
    *out = s;
    return 0;
}

extern "C" void mpb_site_list_destroy(mpb_site_list* s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    delete s;
}

extern "C" int mpb_site_list_seal(mpb_site_list* s, int64_t* n_sites) {
    if (!s || !n_sites) return fail(MPB_EINVAL, "NULL argument");
    if (s->sealed) return fail(MPB_EINVAL, "the site list is sealed already");
    mpb_ctx* ctx = s->ctx;
    CK(cudaSetDevice(ctx->device));
    s->count.assign(s->n_pat, 0);
    if (s->n > 0) {
        DMem alt, tmp, cnt;
        if (alt.reserve((size_t)s->n * 8) != cudaSuccess) return sites_no_memory("sort buffer", s->n, s->n * 8);
        unsigned long long *a = s->keys.as<unsigned long long>(), *b = alt.as<unsigned long long>();
        const long long n = s->n;
        const int bits = s->pat_bits + s->pos_bits + 4;
        if (int rc = cub_run(ctx, "k_sites_seal", tmp, [&](void* t, size_t& bytes) {
                return cub::DeviceRadixSort::SortKeys(t, bytes, a, b, n, 0, bits, ctx->stream);
            }))
            return rc;
        std::swap(s->keys.p, alt.p);
        std::swap(s->keys.bytes, alt.bytes);
        CK(cnt.reserve((size_t)s->n_pat * 8));
        CK(cudaMemsetAsync(cnt.p, 0, (size_t)s->n_pat * 8, ctx->stream));
        MPB_LAUNCH(ctx, k_sites_count, grid_of(n), 256, 0, s->keys.as<unsigned long long>(), n, s->pat_bits,
                   cnt.as<unsigned long long>());
        CK(cudaMemcpyAsync(s->count.data(), cnt.p, (size_t)s->n_pat * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    s->sealed = true;
    *n_sites = s->n;
    return 0;
}

extern "C" int mpb_site_list_keys(mpb_site_list* s, int64_t cap, uint64_t* keys, int64_t* n_sites) {
    if (!s || !n_sites || (cap > 0 && !keys)) return fail(MPB_EINVAL, "NULL argument");
    *n_sites = s->n;
    const long long k = cap < s->n ? cap : s->n;
    if (k <= 0) return 0;
    CK(cudaSetDevice(s->ctx->device));
    CK(cudaMemcpyAsync(keys, s->keys.p, (size_t)k * 8, cudaMemcpyDeviceToHost, s->ctx->stream));
    CK(cudaStreamSynchronize(s->ctx->stream));
    return 0;
}

static int sites_join_args(const mpb_site_list* s, int32_t lo, int32_t hi) {
    if (!s->sealed) return fail(MPB_EINVAL, "the site list is not sealed");
    if (lo < 1 || lo > hi) return fail(MPB_EINVAL, "product lengths %d..%d: need 0 < lo <= hi", lo, hi);
    return 0;
}

extern "C" int mpb_sites_cross(mpb_site_list* s, int32_t lo, int32_t hi, int32_t pair, const uint32_t* eligible,
                               uint8_t* bits) {
    if (!s || !eligible || !bits) return fail(MPB_EINVAL, "NULL argument");
    if (int rc = sites_join_args(s, lo, hi)) return rc;
    const int n_pairs = s->n_pat / 4, words = (n_pairs + 31) / 32;
    if (pair < 0 || pair >= n_pairs) return fail(MPB_EINVAL, "pair %d outside 0..%d", pair, n_pairs - 1);
    memset(bits, 0, n_pairs);
    long long n_pick = 0;
    for (int p = 4 * pair; p < 4 * pair + 4; ++p) n_pick += s->count[p];
    if (n_pick == 0) return 0;
    mpb_ctx* ctx = s->ctx;
    CK(cudaSetDevice(ctx->device));
    DMem d_pick, d_n, d_elig, d_out;
    if (d_pick.reserve((size_t)n_pick * 8) != cudaSuccess) return sites_no_memory("pick", n_pick, n_pick * 8);
    CK(d_n.reserve(8));
    CK(d_elig.reserve((size_t)words * 4));
    CK(d_out.reserve((size_t)(n_pairs + 3) / 4 * 4));
    CK(cudaMemsetAsync(d_n.p, 0, 8, ctx->stream));
    CK(cudaMemsetAsync(d_out.p, 0, (size_t)(n_pairs + 3) / 4 * 4, ctx->stream));
    CK(cudaMemcpyAsync(d_elig.p, eligible, (size_t)words * 4, cudaMemcpyHostToDevice, ctx->stream));
    MPB_LAUNCH(ctx, k_sites_pick, grid_of(s->n), 256, 0, s->keys.as<unsigned long long>(), (long long)s->n, s->pat_bits,
               4 * pair, d_pick.as<long long>(), d_n.as<unsigned long long>());
    MPB_LAUNCH(ctx, k_sites_cross, (unsigned)((n_pick + CROSS_WARPS - 1) / CROSS_WARPS), CROSS_WARPS * 32,
               (size_t)words * 4, s->keys.as<unsigned long long>(), (long long)s->n, d_pick.as<long long>(), n_pick,
               s->pat_bits, s->d_lens.as<int32_t>(), s->d_off.as<int64_t>(), s->d_len.as<int64_t>(), (int)s->n_rec,
               (int)lo, (int)hi, d_elig.as<uint32_t>(), words, d_out.as<uint32_t>());
    CK(cudaMemcpyAsync(bits, d_out.p, n_pairs, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int mpb_sites_own(mpb_site_list* s, int32_t lo, int32_t hi, uint8_t* bits) {
    if (!s || !bits) return fail(MPB_EINVAL, "NULL argument");
    if (int rc = sites_join_args(s, lo, hi)) return rc;
    const int n_pairs = s->n_pat / 4;
    memset(bits, 0, n_pairs);
    if (s->n == 0) return 0;
    mpb_ctx* ctx = s->ctx;
    CK(cudaSetDevice(ctx->device));
    const long long n = s->n;
    DMem k1, k2, tmp, d_out;
    if (k1.reserve((size_t)n * 8) != cudaSuccess || k2.reserve((size_t)n * 8) != cudaSuccess)
        return sites_no_memory("pattern-first copy", n, 2 * n * 8);
    CK(d_out.reserve((size_t)(n_pairs + 3) / 4 * 4));
    CK(cudaMemsetAsync(d_out.p, 0, (size_t)(n_pairs + 3) / 4 * 4, ctx->stream));
    unsigned long long *a = k1.as<unsigned long long>(), *b = k2.as<unsigned long long>();
    MPB_LAUNCH(ctx, k_sites_repack, grid_of(n), 256, 0, s->keys.as<unsigned long long>(), n, s->pat_bits, s->pos_bits, a);
    const int key_bits = s->pat_bits + s->pos_bits + 4;
    if (int rc = cub_run(ctx, "k_sites_own_sort", tmp, [&](void* t, size_t& bytes) {
            return cub::DeviceRadixSort::SortKeys(t, bytes, a, b, n, 0, key_bits, ctx->stream);
        }))
        return rc;
    MPB_LAUNCH(ctx, k_sites_own, grid_of(n), 256, 0, b, n, s->pos_bits, s->d_lens.as<int32_t>(), s->d_off.as<int64_t>(),
               s->d_len.as<int64_t>(), (int)s->n_rec, (int)lo, (int)hi, d_out.as<uint32_t>());
    CK(cudaMemcpyAsync(bits, d_out.p, n_pairs, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}
