// mpb_pools.cu — mpb_pool_search: split n primer pairs into P balanced pools with the least conflict weight inside the
// pools, by independent restarts of a tabu search (multiprime_b200/primer_pools.py states the rule step by step; the
// CPU double tests/fake_pool_search.py restates it and the GPU tests compare the two restart by restart).
//
// One CTA per restart (grid-striding over the restarts).  Shared memory holds D[a][p] = sum of w(a, b) over the pairs b
// in pool p and the tabu table, n*P int32 each (64 KB each at 512 x 32); w (n*n bytes, <= 256 KB) is read through L1/L2,
// one row at a time, so the candidate loop reads it coalesced.  Each step compacts the conflicting pairs, strides the
// candidates over the threads, takes the block minimum of a packed (biased delta, candidate index) key, and updates D
// with one thread per pair.  The result of a restart depends only on (w, P, seed, restart, iterations).
#include "mpb_host.h"

#define POOL_THREADS 512
#define POOL_MAX_N 512
#define POOL_MAX_P 32
#define POOL_MAX_RESTARTS (1ll << 24)
#define POOL_MAX_ITER ((1 << 20) - 1)
#define POOL_BIAS (1 << 24)  // |delta| <= 4 * 255 * 511 + 2 * 255 < 2^20
#define POOL_NONE 0xFFFFFFFFFFFFFFFFull

// splitmix64's finaliser on the packed counter (restart << 40 | step << 20 | slot), keyed by the finalised seed
__host__ __device__ static inline uint64_t pool_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__host__ __device__ static inline uint64_t pool_hash(uint64_t seed, uint64_t restart, uint64_t step, uint64_t slot) {
    return pool_mix(pool_mix(seed) ^ ((restart << 40) | (step << 20) | slot));
}

static inline size_t pool_smem_bytes(int n, int P) {
    return (size_t)n * P * 4 * 2 + (size_t)n * 2 + (size_t)n + 16;
}

__global__ void __launch_bounds__(POOL_THREADS)
k_pool_search(const uint8_t* __restrict__ w, int n, int P, uint64_t seed, int64_t r0, int64_t nr, int iters,
              long long* __restrict__ best_cost, int32_t* __restrict__ best_step, uint8_t* __restrict__ assign) {
    extern __shared__ int32_t sm[];
    int32_t* D = sm;                              // [n][P]
    int32_t* tabu = D + n * P;                    // [n][P]: a pair may return to pool p from step tabu[a][p] on
    int16_t* conf = (int16_t*)(tabu + n * P);     // [n]: the shuffle, then the conflicting pairs of a step
    uint8_t* pool = (uint8_t*)(conf + n);         // [n]
    __shared__ int s_size[POOL_MAX_P];
    __shared__ int s_nconf, s_cost;
    __shared__ unsigned long long s_red[POOL_THREADS / 32];
    __shared__ unsigned long long s_key;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int hi = (n + P - 1) / P, lo = n / P;
    const bool moves = (n % P) != 0;
    // the swap candidates c = k * n + b (k-th conflicting pair, partner b), walked without a division per step
    const int k_stride = nt / n, b_stride = nt % n;

    for (int64_t ri = blockIdx.x; ri < nr; ri += gridDim.x) {
        const uint64_t r = (uint64_t)(r0 + ri);
        // -- start: Fisher-Yates shuffle of the pairs, the k-th of the shuffle to pool k mod P --------------------
        if (tid == 0) {
            for (int k = 0; k < n; ++k) conf[k] = (int16_t)k;
            for (int k = n - 1; k > 0; --k) {
                const int j = (int)(pool_hash(seed, r, 0, (uint64_t)k) % (uint64_t)(k + 1));
                const int16_t t = conf[k];
                conf[k] = conf[j];
                conf[j] = t;
            }
            s_cost = 0;
        }
        for (int p = tid; p < P; p += nt) s_size[p] = lo + (p < n % P ? 1 : 0);
        __syncthreads();
        for (int k = tid; k < n; k += nt) pool[conf[k]] = (uint8_t)(k % P);
        __syncthreads();
        int part = 0;
        for (int a = tid; a < n; a += nt) {
            int32_t* Da = D + a * P;
            for (int p = 0; p < P; ++p) {
                Da[p] = 0;
                tabu[a * P + p] = 0;
            }
            const uint8_t* wa = w + (size_t)a * n;
            for (int b = 0; b < n; ++b) Da[pool[b]] += __ldg(wa + b);
            part += Da[pool[a]];
            assign[(size_t)ri * n + a] = pool[a];
        }
        if (part) atomicAdd(&s_cost, part);
        __syncthreads();
        int cost = s_cost / 2, best = cost, best_t = 0;

        // -- steps --------------------------------------------------------------------------------------------
        for (int t = 1; t <= iters && cost > 0; ++t) {
            if (tid == 0) s_nconf = 0;
            __syncthreads();
            for (int a = tid; a < n; a += nt)
                if (D[a * P + pool[a]] > 0) conf[atomicAdd(&s_nconf, 1)] = (int16_t)a;
            __syncthreads();
            const int K = s_nconf;
            unsigned long long key = POOL_NONE;
            int k = tid / n, b = tid % n;
            for (; k < K; k += k_stride, b += b_stride) {
                if (b >= n) {
                    b -= n;
                    ++k;
                    if (k >= K) break;
                }
                const int a = conf[k], pa = pool[a], pb = pool[b];
                if (pa == pb) continue;
                const int delta = D[a * P + pb] - D[a * P + pa] + D[b * P + pa] - D[b * P + pb] -
                                  2 * (int)__ldg(w + (size_t)a * n + b);
                const bool is_tabu = tabu[a * P + pb] > t || tabu[b * P + pa] > t;
                if (is_tabu && cost + delta >= best) continue;
                const unsigned long long c = ((unsigned long long)(delta + POOL_BIAS) << 32) | (unsigned)(a * n + b);
                key = c < key ? c : key;
            }
            if (moves) {
                for (int c = tid; c < K * P; c += nt) {
                    const int a = conf[c / P], q = c % P, pa = pool[a];
                    if (s_size[pa] != hi || s_size[q] != lo) continue;
                    const int delta = D[a * P + q] - D[a * P + pa];
                    if (tabu[a * P + q] > t && cost + delta >= best) continue;
                    const unsigned long long cc =
                        ((unsigned long long)(delta + POOL_BIAS) << 32) | (unsigned)(n * n + a * P + q);
                    key = cc < key ? cc : key;
                }
            }
            for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long x = __shfl_xor_sync(0xffffffffu, key, o);
                key = x < key ? x : key;
            }
            if ((tid & 31) == 0) s_red[tid >> 5] = key;
            __syncthreads();
            if (tid < 32) {
                key = tid < (nt >> 5) ? s_red[tid] : POOL_NONE;
                for (int o = 16; o > 0; o >>= 1) {
                    const unsigned long long x = __shfl_xor_sync(0xffffffffu, key, o);
                    key = x < key ? x : key;
                }
                if (tid == 0) s_key = key;
            }
            __syncthreads();
            key = s_key;
            if (key == POOL_NONE) break;                 // no admissible candidate
            const int delta = (int)(key >> 32) - POOL_BIAS;
            const int idx = (int)(unsigned)key;
            const bool is_move = idx >= n * n;
            const int a = is_move ? (idx - n * n) / P : idx / n;
            const int pa = pool[a];
            const int bb = is_move ? -1 : idx % n;
            const int pb = is_move ? (idx - n * n) % P : pool[bb];
            __syncthreads();                             // every thread has read pool[] before it changes
            if (tid == 0) {
                const int tenure = 10 + (6 * K) / 10 + (int)(pool_hash(seed, r, (uint64_t)t, 0) % 10);
                tabu[a * P + pa] = t + tenure;
                pool[a] = (uint8_t)pb;
                if (is_move) {
                    s_size[pa] -= 1;
                    s_size[pb] += 1;
                } else {
                    tabu[bb * P + pb] = t + tenure;
                    pool[bb] = (uint8_t)pa;
                }
            }
            const uint8_t* wa = w + (size_t)a * n;       // w is symmetric: row a is column a
            const uint8_t* wb = w + (size_t)(is_move ? a : bb) * n;
            for (int x = tid; x < n; x += nt) {
                const int wxa = __ldg(wa + x);
                const int wxb = is_move ? 0 : (int)__ldg(wb + x);
                D[x * P + pa] += wxb - wxa;
                D[x * P + pb] += wxa - wxb;
            }
            cost += delta;
            __syncthreads();
            if (cost < best) {
                best = cost;
                best_t = t;
                for (int x = tid; x < n; x += nt) assign[(size_t)ri * n + x] = pool[x];
            }
        }
        if (tid == 0) {
            best_cost[ri] = best;
            best_step[ri] = best_t;
        }
        __syncthreads();                                 // the next restart reuses the shared arrays
    }
}

extern "C" int mpb_pool_search(mpb_ctx* ctx, int32_t n, int32_t n_pools, const uint8_t* w, uint64_t seed, int64_t r0,
                               int64_t r1, int32_t iterations, int64_t* best_cost, int32_t* best_step, uint8_t* assign) {
    if (!ctx || !w || !best_cost || !best_step || !assign) return mpb_fail(MPB_EINVAL, "NULL argument");
    if (n < 1 || n > POOL_MAX_N) return mpb_fail(MPB_EINVAL, "%d pairs: need 1 <= pairs <= %d", n, POOL_MAX_N);
    if (n_pools < 1 || n_pools > POOL_MAX_P)
        return mpb_fail(MPB_EINVAL, "%d pools: need 1 <= pools <= %d", n_pools, POOL_MAX_P);
    if (n_pools > n) return mpb_fail(MPB_EINVAL, "%d pools for %d pairs: need pools <= pairs", n_pools, n);
    if (r0 < 0 || r1 < r0 || r1 > POOL_MAX_RESTARTS)
        return mpb_fail(MPB_EINVAL, "restarts [%lld, %lld): need 0 <= r0 <= r1 <= %lld", (long long)r0, (long long)r1,
                        POOL_MAX_RESTARTS);
    if (iterations < 0 || iterations > POOL_MAX_ITER)
        return mpb_fail(MPB_EINVAL, "%d iterations: need 0 <= iterations <= %d", iterations, POOL_MAX_ITER);
    for (int a = 0; a < n; ++a) {
        if (w[(size_t)a * n + a]) return mpb_fail(MPB_EINVAL, "w[%d][%d] = %d: the diagonal must be zero", a, a,
                                                  (int)w[(size_t)a * n + a]);
        for (int b = a + 1; b < n; ++b)
            if (w[(size_t)a * n + b] != w[(size_t)b * n + a])
                return mpb_fail(MPB_EINVAL, "w is not symmetric: w[%d][%d] = %d, w[%d][%d] = %d", a, b,
                                (int)w[(size_t)a * n + b], b, a, (int)w[(size_t)b * n + a]);
    }
    const int64_t nr = r1 - r0;
    if (nr == 0) return 0;
    MPB_CK(cudaSetDevice(mpb_ctx_device(ctx)));
    cudaStream_t st = mpb_ctx_stream(ctx);
    const size_t smem = pool_smem_bytes(n, n_pools);
    MPB_CK(cudaFuncSetAttribute(k_pool_search, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    MPB_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pool_search, POOL_THREADS, smem));
    const int64_t wave = (int64_t)(per_sm > 0 ? per_sm : 1) * mpb_ctx_sms(ctx);
    const unsigned grid = (unsigned)(nr < wave ? nr : wave);
    uint8_t *dw, *dassign;
    long long* dcost;
    int32_t* dstep;
    MPB_CK(cudaMallocAsync(&dw, (size_t)n * n, st));
    MPB_CK(cudaMallocAsync(&dassign, (size_t)nr * n, st));
    MPB_CK(cudaMallocAsync(&dcost, (size_t)nr * 8, st));
    MPB_CK(cudaMallocAsync(&dstep, (size_t)nr * 4, st));
    MPB_CK(cudaMemcpyAsync(dw, w, (size_t)n * n, cudaMemcpyHostToDevice, st));
    ctx->pending_units = (double)nr;
    MPB_LAUNCH(ctx, k_pool_search, grid, POOL_THREADS, smem, dw, n, n_pools, (uint64_t)seed, r0, nr, iterations, dcost,
               dstep, dassign);
    MPB_CK(cudaMemcpyAsync(best_cost, dcost, (size_t)nr * 8, cudaMemcpyDeviceToHost, st));
    MPB_CK(cudaMemcpyAsync(best_step, dstep, (size_t)nr * 4, cudaMemcpyDeviceToHost, st));
    MPB_CK(cudaMemcpyAsync(assign, dassign, (size_t)nr * n, cudaMemcpyDeviceToHost, st));
    MPB_CK(cudaStreamSynchronize(st));
    cudaFreeAsync(dw, st);
    cudaFreeAsync(dassign, st);
    cudaFreeAsync(dcost, st);
    cudaFreeAsync(dstep, st);
    return 0;
}
