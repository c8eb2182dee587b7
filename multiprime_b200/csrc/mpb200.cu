// mpb200.cu — libmpb200.so: kernels + C ABI (include/mpb200.h) of the H100 degenerate-primer candidate scan.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared -Xcompiler -fPIC (see build.py)
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <algorithm>
#include <vector>

#include "mpb200.h"
#include "mpb_host.h"
#include "mpb_device.cuh"
#include "mpb_prefilter.h"

// ------------------------------------------------------------------------------------------------------
// host-side plumbing (shared pieces live in mpb_host.h)
// ------------------------------------------------------------------------------------------------------
static thread_local std::string g_err;

int mpb_fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define fail mpb_fail
#define CK MPB_CK
#define LAUNCH MPB_LAUNCH

int mpb_check_flags(mpb_ctx* ctx, int* dflags) {
    int f = 0;
    CK(cudaMemcpyAsync(&f, dflags, sizeof f, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (f) {
        int zero = 0;
        cudaMemcpyAsync(dflags, &zero, sizeof zero, cudaMemcpyHostToDevice, ctx->stream);
    }
    if (f & MPB_ERR_TABLE_FULL) return fail(MPB_EOVERFLOW, "haplotype table full: rebuild with a larger log2_cap");
    if (f & MPB_ERR_EXPAND)
        return fail(MPB_EEXPAND, "a window of one sequence expands to more than %u haplotypes", MPB_MAX_EXP);
    if (f & MPB_ERR_SHORT_ROW) return fail(MPB_EEXPAND, "a sequence holds fewer than k bases");
    return 0;
}

extern "C" int mpb_abi_version(void) { return MPB_ABI_VERSION; }
extern "C" const char* mpb_last_error(void) { return g_err.c_str(); }
extern "C" int mpb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" int mpb_ctx_create(int device, mpb_ctx** out) {
    if (!out) return fail(MPB_EINVAL, "out is NULL");
    int n = mpb_device_count();
    if (n == 0) return fail(MPB_ECUDA, "no CUDA device: libmpb200 has no CPU fallback");
    if (device < 0 || device >= n) return fail(MPB_EINVAL, "device %d out of range (0..%d)", device, n - 1);
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(MPB_ECUDA, "device %d is sm_%d%d; libmpb200 is built for sm_90a (H100) only", device, prop.major,
                    prop.minor);
    cudaMemPool_t pool;
    CK(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t thr = UINT64_MAX;
    CK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    mpb_ctx* c = new mpb_ctx;
    c->device = device;
    c->stream = 0;
    c->launches = 0;
    c->sm_count = prop.multiProcessorCount;
    c->profile = false;
    c->pending_units = 0;
    c->copy_stream = nullptr;
    c->pinned = nullptr;
    if (cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaMallocHost(&c->pinned, MPB_CTX_PINNED_INTS * sizeof(int)) != cudaSuccess) {
        if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
        delete c;
        return fail(MPB_ECUDA, "copy stream / pinned scratch");
    }
    *out = c;
    return 0;
}
extern "C" void mpb_ctx_destroy(mpb_ctx* ctx) {
    if (!ctx) return;
    for (auto& r : ctx->recs) {
        cudaEventDestroy(r.e0);
        cudaEventDestroy(r.e1);
    }
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    delete ctx;
}
extern "C" int mpb_ctx_set_stream(mpb_ctx* ctx, void* s) {
    if (!ctx) return fail(MPB_EINVAL, "ctx is NULL");
    ctx->stream = (cudaStream_t)s;
    return 0;
}
extern "C" int mpb_ctx_sync(mpb_ctx* ctx) {
    if (!ctx) return fail(MPB_EINVAL, "ctx is NULL");
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}
extern "C" int64_t mpb_ctx_launches(mpb_ctx* ctx) { return ctx ? ctx->launches : 0; }

// stream-ordered device memory for results that stay in HBM between calls (bit vectors of the scan -> pair coverage)
extern "C" int mpb_dev_alloc(mpb_ctx* ctx, int64_t bytes, void** out) {
    if (!ctx || !out || bytes < 0) return fail(MPB_EINVAL, "bad argument");
    CK(cudaSetDevice(ctx->device));
    void* p = nullptr;
    cudaError_t e = cudaMallocAsync(&p, bytes > 0 ? (size_t)bytes : 1, ctx->stream);
    if (e != cudaSuccess) return fail(MPB_ENOMEM, "%lld bytes: %s", (long long)bytes, cudaGetErrorString(e));
    *out = p;
    return 0;
}
extern "C" void mpb_dev_free(mpb_ctx* ctx, void* p) {
    if (ctx && p) cudaFreeAsync(p, ctx->stream);
}

// plain copy between any two of host / device memory on the context's stream, synchronised on return
extern "C" int mpb_ctx_memcpy(mpb_ctx* ctx, void* dst, const void* src, int64_t bytes) {
    if (!ctx || !dst || !src || bytes < 0) return fail(MPB_EINVAL, "bad argument");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int mpb_ctx_memset(mpb_ctx* ctx, void* dst, int value, int64_t bytes) {
    if (!ctx || !dst || bytes < 0) return fail(MPB_EINVAL, "bad argument");
    if (!mpb_is_device_ptr(dst)) return fail(MPB_EINVAL, "dst must be device memory");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemsetAsync(dst, value, (size_t)bytes, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int mpb_ctx_profile(mpb_ctx* ctx, int enable) {
    if (!ctx) return fail(MPB_EINVAL, "ctx is NULL");
    ctx->profile = enable != 0;
    return 0;
}

// Sum the event-timed durations of all launches of `kernel` recorded since the last read; clears them when
// kernel is NULL.  ms / launches / units may be NULL.
extern "C" int mpb_ctx_profile_read(mpb_ctx* ctx, const char* kernel, double* ms, int64_t* launches, double* units) {
    if (!ctx) return fail(MPB_EINVAL, "ctx is NULL");
    CK(cudaStreamSynchronize(ctx->stream));
    if (!kernel) {
        for (auto& r : ctx->recs) {
            cudaEventDestroy(r.e0);
            cudaEventDestroy(r.e1);
        }
        ctx->recs.clear();
        ctx->extra_units.clear();
        return 0;
    }
    double t = 0, u = 0;
    {
        auto it = ctx->extra_units.find(kernel);  // units counted on the device (candidates of the resident walk)
        if (it != ctx->extra_units.end()) u += it->second;
    }
    int64_t n = 0;
    for (auto& r : ctx->recs)
        if (strncmp(r.name, kernel, strlen(kernel)) == 0 && (r.name[strlen(kernel)] == 0 || r.name[strlen(kernel)] == '<')) {
            float f = 0;
            CK(cudaEventElapsedTime(&f, r.e0, r.e1));
            t += f;
            u += r.units;
            ++n;
        }
    if (ms) *ms = t;
    if (launches) *launches = n;
    if (units) *units = u;
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// alignment upload: nibble rows -> bit-planes
// ------------------------------------------------------------------------------------------------------
// nibble rows -> row planes.  A block stages PACK_ROWS rows x PACK_SEG bytes (512 columns) through shared memory so
// that the global reads are contiguous pieces of each row (the first version read 16 B at a row stride per thread);
// thread = (row, column word), rows fastest, so the uint4 plane stores coalesce too.
#define PACK_ROWS 64
#define PACK_SEG 256
__global__ void __launch_bounds__(256)
k_pack_planes(const uint8_t* __restrict__ packed, int64_t row_first, int64_t n_rows, int64_t n_seq, int64_t nsp,
              int64_t row_bytes, const int32_t* __restrict__ lens, int ncw, uint32_t* __restrict__ planes) {
    __shared__ __align__(16) uint8_t tile[PACK_ROWS][PACK_SEG + 4];
    const int64_t r0 = (int64_t)blockIdx.x * PACK_ROWS;  // relative to row_first
    const int64_t seg0 = (int64_t)blockIdx.y * PACK_SEG;
    for (int i = threadIdx.x; i < PACK_ROWS * PACK_SEG; i += 256) {
        const int r = i / PACK_SEG, b = i % PACK_SEG;
        const int64_t s = row_first + r0 + r;
        uint8_t x = 0;
        if (r0 + r < n_rows && s < n_seq && seg0 + b < row_bytes) x = packed[(r0 + r) * row_bytes + seg0 + b];
        tile[r][b] = x;
    }
    __syncthreads();
    const int r = threadIdx.x & (PACK_ROWS - 1);
    const int64_t s = row_first + r0 + r;
    if (r0 + r >= n_rows || s >= nsp) return;
    const int len = s < n_seq ? lens[s] : 0;
    for (int cwl = threadIdx.x / PACK_ROWS; cwl < PACK_SEG / 16; cwl += 256 / PACK_ROWS) {
        const int cw = blockIdx.y * (PACK_SEG / 16) + cwl;
        if (cw >= ncw) break;
        uint32_t a = 0, c = 0, g = 0, t = 0;
        const int col0 = cw * 32;
        if (cw < ncw - 1) {
            for (int i = 0; i < 32; i += 2) {
                const int col = col0 + i;
                if (col >= len) break;
                const uint32_t b = tile[r][cwl * 16 + (i >> 1)];
                const uint32_t x = b & 15u;
                const uint32_t y = (col + 1 < len) ? (b >> 4) : 0u;
                a |= ((x & 1u) << i) | ((y & 1u) << (i + 1));
                c |= (((x >> 1) & 1u) << i) | (((y >> 1) & 1u) << (i + 1));
                g |= (((x >> 2) & 1u) << i) | (((y >> 2) & 1u) << (i + 1));
                t |= (((x >> 3) & 1u) << i) | (((y >> 3) & 1u) << (i + 1));
            }
        }
        reinterpret_cast<uint4*>(planes)[(int64_t)cw * nsp + s] = make_uint4(a, c, g, t);
    }
}

// row planes -> column view: a 32 x 32 bit transpose per (column word, 32-sequence word, base).  Block = 32 warps =
// 32 consecutive sequence words of one column word; warp: lane = sequence, one ballot per (base, column); the 32 x 4
// x 32 result words go through shared memory so that every column-plane row is written in 128-byte pieces.
__global__ void __launch_bounds__(1024)
k_build_colp(const uint32_t* __restrict__ planes, int64_t nsp, int64_t nwords, int64_t word_first, int64_t n_words_chunk,
             uint32_t* __restrict__ colp) {
    __shared__ uint32_t tile[32 * 4][33];
    const int cw = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t w = word_first + (int64_t)blockIdx.x * 32 + warp;
    const bool live = (int64_t)blockIdx.x * 32 + warp < n_words_chunk && w < nwords;
    uint4 q = make_uint4(0, 0, 0, 0);
    if (live) q = __ldg(reinterpret_cast<const uint4*>(planes) + (int64_t)cw * nsp + w * 32 + lane);
#pragma unroll 4
    for (int c = 0; c < 32; ++c) {
        const unsigned ba = __ballot_sync(0xffffffffu, (q.x >> c) & 1u), bc = __ballot_sync(0xffffffffu, (q.y >> c) & 1u),
                       bg = __ballot_sync(0xffffffffu, (q.z >> c) & 1u), bt = __ballot_sync(0xffffffffu, (q.w >> c) & 1u);
        if (lane == 0) {
            tile[c * 4 + 0][warp] = ba;
            tile[c * 4 + 1][warp] = bc;
            tile[c * 4 + 2][warp] = bg;
            tile[c * 4 + 3][warp] = bt;
        }
    }
    __syncthreads();
    // thread (row = c*4 + b, word): 128 rows x 32 words = 4 per thread
    for (int i = threadIdx.x; i < 128 * 32; i += 1024) {
        const int row = i >> 5, ww = i & 31;
        const int64_t wo = word_first + (int64_t)blockIdx.x * 32 + ww;
        if ((int64_t)blockIdx.x * 32 + ww < n_words_chunk && wo < nwords)
            colp[((int64_t)cw * 128 + row) * nwords + wo] = tile[row][ww];
    }
}

__global__ void k_fill_u32(uint32_t* __restrict__ dst, int64_t n, uint32_t value) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = value;
}

__global__ void k_fill_i32(int32_t* __restrict__ dst, int64_t n, int64_t n_set, int32_t value) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = i < n_set ? value : 0;
}

// a frequent base of every column, counted on up to CONS_SAMPLE 32-sequence words spread evenly over the rows
#define CONS_SAMPLE 1024
__global__ void __launch_bounds__(128)
k_col_consensus(const uint32_t* __restrict__ colp, int64_t nwords, uint8_t* __restrict__ cons) {
    __shared__ unsigned int s_n[4];
    if (threadIdx.x < 4) s_n[threadIdx.x] = 0;
    __syncthreads();
    const int col = blockIdx.x;
    const int64_t n_s = nwords < CONS_SAMPLE ? nwords : CONS_SAMPLE;
    unsigned n[4] = {0, 0, 0, 0};
    for (int64_t i = threadIdx.x; i < n_s; i += 128) {
        const int64_t w = i * nwords / n_s;
#pragma unroll
        for (int b = 0; b < 4; ++b) n[b] += __popc(__ldg(colp + ((int64_t)col * 4 + b) * nwords + w));
    }
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        const unsigned t = __reduce_add_sync(0xffffffffu, n[b]);
        if ((threadIdx.x & 31) == 0) atomicAdd(&s_n[b], t);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int best = 0;
        for (int b = 1; b < 4; ++b)
            if (s_n[b] > s_n[best]) best = b;
        cons[col] = (uint8_t)best;
    }
}

#define UPLOAD_CHUNK_ROWS 65536  // multiple of 1024 (k_build_colp tiles) and of PACK_ROWS

extern "C" int mpb_msa_upload(mpb_ctx* ctx, const uint8_t* packed4, int64_t n_seq, int64_t n_col, int64_t row_bytes,
                              const int32_t* lens, mpb_msa** out) {
    if (!ctx || !packed4 || !out) return fail(MPB_EINVAL, "NULL argument");
    if (n_seq < 1 || n_col < 1 || row_bytes < (n_col + 1) / 2)
        return fail(MPB_EINVAL, "bad shape n_seq=%lld n_col=%lld row_bytes=%lld", (long long)n_seq, (long long)n_col,
                    (long long)row_bytes);
    if (n_seq >= (1ll << 31)) return fail(MPB_EINVAL, "n_seq must be < 2^31");
    // k_build_colp puts one 32-column word per blockIdx.y
    if ((n_col + 31) / 32 > 65535)
        return fail(MPB_EINVAL, "n_col=%lld: at most 65535 x 32 = 2097120 columns are supported", (long long)n_col);
    CK(cudaSetDevice(ctx->device));
    mpb_msa* m = new mpb_msa;
    memset(m, 0, sizeof *m);
    m->ctx = ctx;
    m->n_seq = n_seq;
    m->nsp = (n_seq + 127) / 128 * 128;
    m->nwords = m->nsp / 32;
    m->n_col = n_col;
    m->ncw = (int)((n_col + 31) / 32) + 1;
    const size_t pbytes = (size_t)m->ncw * 4 * m->nsp * sizeof(uint32_t);
    const size_t crows = (size_t)(m->ncw - 1) * 128 + 2;
    cudaError_t e = cudaMallocAsync(&m->planes, pbytes, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&m->colp, crows * m->nwords * 4, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&m->lens, m->nsp * sizeof(int32_t), ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&m->err, sizeof(int), ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&m->cons, (size_t)(m->ncw - 1) * 32, ctx->stream);
    if (e != cudaSuccess) {
        mpb_msa_free(m);
        return fail(MPB_ENOMEM, "alignment planes (2 x %zu bytes): %s", pbytes, cudaGetErrorString(e));
    }
    CK(cudaMemsetAsync(m->err, 0, sizeof(int), ctx->stream));
    std::vector<int32_t> hl;
    if (lens) {
        hl.assign(m->nsp, 0);
        for (int64_t i = 0; i < n_seq; ++i) {
            if (lens[i] < 0 || lens[i] > n_col) {
                mpb_msa_free(m);
                return fail(MPB_EINVAL, "lens[%lld]=%d outside 0..n_col", (long long)i, lens[i]);
            }
            hl[i] = lens[i];
            if (lens[i] < n_col) m->short_rows = true;
        }
        CK(cudaMemcpyAsync(m->lens, hl.data(), m->nsp * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    } else {
        LAUNCH(ctx, k_fill_i32, (unsigned)((m->nsp + 255) / 256), 256, 0, m->lens, m->nsp, n_seq, (int32_t)n_col);
    }
    LAUNCH(ctx, k_fill_u32, (unsigned)((m->nwords + 255) / 256), 256, 0, m->colp + (size_t)MPB_COLP_ONES(m) * m->nwords,
           m->nwords, 0xFFFFFFFFu);
    LAUNCH(ctx, k_fill_u32, (unsigned)((m->nwords + 255) / 256), 256, 0, m->colp + (size_t)MPB_COLP_ZEROS(m) * m->nwords,
           m->nwords, 0u);
    // rows travel in chunks: the H2D copy of chunk i+1 (copy stream) overlaps the plane / column-view build of chunk i
    const bool on_dev = mpb_is_device_ptr(packed4);
    const int64_t chunk = UPLOAD_CHUNK_ROWS;
    uint8_t* stage[2] = {nullptr, nullptr};
    cudaEvent_t copied[2] = {nullptr, nullptr}, consumed[2] = {nullptr, nullptr};
    int rc = 0;
    if (!on_dev) {
        const size_t sb = (size_t)(n_seq < chunk ? n_seq : chunk) * row_bytes;
        for (int i = 0; i < 2 && rc == 0; ++i) {
            if (cudaMallocAsync(&stage[i], sb, ctx->stream) != cudaSuccess || cudaEventCreateWithFlags(&copied[i], cudaEventDisableTiming) != cudaSuccess ||
                cudaEventCreateWithFlags(&consumed[i], cudaEventDisableTiming) != cudaSuccess)
                rc = fail(MPB_ENOMEM, "upload staging buffers");
        }
        if (rc == 0 && cudaEventRecord(consumed[0], ctx->stream) != cudaSuccess) rc = fail(MPB_ECUDA, "event record");
        if (rc == 0 && cudaEventRecord(consumed[1], ctx->stream) != cudaSuccess) rc = fail(MPB_ECUDA, "event record");
    }
    int slot = 0;
    for (int64_t r0 = 0; r0 < m->nsp && rc == 0; r0 += chunk, slot ^= 1) {
        const int64_t rows = (m->nsp - r0 < chunk) ? m->nsp - r0 : chunk;          // plane rows (incl. padding rows)
        const int64_t src_rows = r0 >= n_seq ? 0 : ((n_seq - r0 < chunk) ? n_seq - r0 : chunk);
        const uint8_t* src = packed4 + r0 * row_bytes;
        if (!on_dev && src_rows > 0) {
            cudaError_t ce = cudaStreamWaitEvent(ctx->copy_stream, consumed[slot], 0);  // staging slot free again
            if (ce == cudaSuccess)
                ce = cudaMemcpyAsync(stage[slot], src, (size_t)src_rows * row_bytes, cudaMemcpyHostToDevice, ctx->copy_stream);
            if (ce == cudaSuccess) ce = cudaEventRecord(copied[slot], ctx->copy_stream);
            if (ce == cudaSuccess) ce = cudaStreamWaitEvent(ctx->stream, copied[slot], 0);
            if (ce != cudaSuccess) {
                rc = fail(MPB_ECUDA, "upload chunk: %s", cudaGetErrorString(ce));
                break;
            }
            src = stage[slot];
        }
        dim3 grid((unsigned)((rows + PACK_ROWS - 1) / PACK_ROWS), (unsigned)((m->ncw * 16 + PACK_SEG - 1) / PACK_SEG));
        k_pack_planes<<<grid, 256, 0, ctx->stream>>>(src, r0, rows, n_seq, m->nsp, row_bytes, m->lens, m->ncw, m->planes);
        ctx->launches++;
        dim3 g2((unsigned)((rows / 32 + 31) / 32), (unsigned)(m->ncw - 1));
        k_build_colp<<<g2, 1024, 0, ctx->stream>>>(m->planes, m->nsp, m->nwords, r0 / 32, rows / 32, m->colp);
        ctx->launches++;
        if (cudaGetLastError() != cudaSuccess) rc = fail(MPB_ECUDA, "upload kernels");
        if (!on_dev && rc == 0 && cudaEventRecord(consumed[slot], ctx->stream) != cudaSuccess) rc = fail(MPB_ECUDA, "event record");
    }
    if (rc == 0) {
        k_col_consensus<<<(unsigned)((m->ncw - 1) * 32), 128, 0, ctx->stream>>>(m->colp, m->nwords, m->cons);
        ctx->launches++;
        if (cudaGetLastError() != cudaSuccess) rc = fail(MPB_ECUDA, "upload kernels");
    }
    cudaError_t se = cudaStreamSynchronize(ctx->stream);  // hl / staging lifetime
    for (int i = 0; i < 2; ++i) {
        if (stage[i]) cudaFreeAsync(stage[i], ctx->stream);
        if (copied[i]) cudaEventDestroy(copied[i]);
        if (consumed[i]) cudaEventDestroy(consumed[i]);
    }
    if (rc == 0 && se != cudaSuccess) rc = fail(MPB_ECUDA, "upload: %s", cudaGetErrorString(se));
    if (rc) {
        mpb_msa_free(m);
        return rc;
    }
    *out = m;
    return 0;
}

extern "C" void mpb_msa_free(mpb_msa* m) {
    if (!m) return;
    if (m->planes) cudaFreeAsync(m->planes, m->ctx->stream);
    if (m->colp) cudaFreeAsync(m->colp, m->ctx->stream);
    if (m->lens) cudaFreeAsync(m->lens, m->ctx->stream);
    if (m->err) cudaFreeAsync(m->err, m->ctx->stream);
    if (m->cons) cudaFreeAsync(m->cons, m->ctx->stream);
    delete m;
}
extern "C" int64_t mpb_msa_nseq(const mpb_msa* m) { return m ? m->n_seq : 0; }
extern "C" int mpb_msa_set_row0(mpb_msa* m, int64_t row0) {
    if (!m || row0 < 0 || row0 + m->n_seq >= (1ll << 47)) return fail(MPB_EINVAL, "bad row0");
    m->row0 = row0;
    return 0;
}

// core:625-627: leading gap count and length without trailing gaps, per sequence
__global__ void k_seq_attr(const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq, const int32_t* __restrict__ lens,
                           int ncw, int32_t* __restrict__ lead, int32_t* __restrict__ rstrip) {
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seq) return;
    int len = lens[s];
    int first = -1, last = -1;
    for (int cw = 0; cw < ncw - 1; ++cw) {
        const uint4 w = mpb_word(pl, nsp, s, cw);
        uint32_t any = w.x | w.y | w.z | w.w;
        if (any) {
            if (first < 0) first = cw * 32 + __ffs(any) - 1;
            last = cw * 32 + 31 - __clz(any);
        }
    }
    lead[s] = first < 0 ? len : first;
    rstrip[s] = last + 1;
}

// histograms of the two per-sequence attributes (values 0..n_col): the host takes the quantiles of core:629-633 from
// the cumulative counts (an order statistic needs no sort), and sequence shards simply add their histograms
__global__ void k_seq_attr_hist(const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq,
                                const int32_t* __restrict__ lens, int ncw, unsigned long long* __restrict__ lead_hist,
                                unsigned long long* __restrict__ rstrip_hist) {
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seq) return;
    int len = lens[s];
    int first = -1, last = -1;
    for (int cw = 0; cw < ncw - 1; ++cw) {
        const uint4 w = mpb_word(pl, nsp, s, cw);
        uint32_t any = w.x | w.y | w.z | w.w;
        if (any) {
            if (first < 0) first = cw * 32 + __ffs(any) - 1;
            last = cw * 32 + 31 - __clz(any);
        }
    }
    const int lead = first < 0 ? len : first, rs = last + 1;
    // warp-aggregate equal values before the atomics (most sequences share the value)
    unsigned peers = __match_any_sync(__activemask(), lead);
    if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&lead_hist[lead], (unsigned long long)__popc(peers));
    peers = __match_any_sync(__activemask(), rs);
    if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&rstrip_hist[rs], (unsigned long long)__popc(peers));
}

extern "C" int mpb_seq_attr_hist(mpb_msa* m, int64_t* lead_hist_hd, int64_t* rstrip_hist_hd) {
    if (!m || !lead_hist_hd || !rstrip_hist_hd) return fail(MPB_EINVAL, "NULL argument");
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    const size_t bytes = (size_t)(m->n_col + 1) * 8;
    OutBuf a(ctx, lead_hist_hd, bytes), b(ctx, rstrip_hist_hd, bytes);
    if (a.rc || b.rc) return MPB_ENOMEM;
    CK(cudaMemsetAsync(a.d, 0, bytes, ctx->stream));
    CK(cudaMemsetAsync(b.d, 0, bytes, ctx->stream));
    LAUNCH(ctx, k_seq_attr_hist, (unsigned)((m->n_seq + 255) / 256), 256, 0, m->planes, m->nsp, m->n_seq, m->lens, m->ncw,
           a.dev<unsigned long long>(), b.dev<unsigned long long>());
    CK(a.finish());
    CK(b.finish());
    if (a.is_host() || b.is_host()) CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int mpb_seq_attr(mpb_msa* m, int32_t* lead_hd, int32_t* rstrip_hd) {
    if (!m || !lead_hd || !rstrip_hd) return fail(MPB_EINVAL, "NULL argument");
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    OutBuf lead(ctx, lead_hd, m->n_seq * sizeof(int32_t)), rs(ctx, rstrip_hd, m->n_seq * sizeof(int32_t));
    if (lead.rc || rs.rc) return lead.rc ? lead.rc : rs.rc;
    LAUNCH(ctx, k_seq_attr, (unsigned)((m->n_seq + 255) / 256), 256, 0, m->planes, m->nsp, m->n_seq, m->lens, m->ncw,
           lead.dev<int32_t>(), rs.dev<int32_t>());
    CK(lead.finish());
    CK(rs.finish());
    if (lead.is_host() || rs.is_host()) CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// window passes: every (window, sequence) k-mer of a window batch, once for the entropy prefilter (all windows) and once
// for the haplotype tables (the windows that survive it)
// ------------------------------------------------------------------------------------------------------
// Both kernels stream without block barriers and read every alignment word ONCE per group of windows.
//   * Windows are grouped by column word (mpb_window_groups: consecutive batch entries with the same p >> 5, at most
//     32): all of them cut their k-mers out of the same two 128-bit plane words of a sequence, so a thread loads the
//     two words once per tile and funnel-shifts up to 32 windows out of them (round 1 and the first version of this
//     round re-read them per window, many GB of L2 traffic per pass).
//   * Block (x, y) owns WIN_TILES x 256 sequences and walks the groups y, y + gridDim.y, ...; a warp owns 32
//     sequences per tile, and LANE j of the warp keeps the running state of WINDOW j of the group.  In a window below
//     the entropy gate most sequences carry the SAME k-mer, so the warp keeps that majority k-mer and its count in
//     lane j's registers for the whole pass (one global atomic per warp and window) and sends only the minority rows
//     to global memory one by one; a variable window degenerates to one atomic per row, which is what it costs
//     anyway.  (Round 1 staged every row in a block-private hash table: three block barriers per window, 150
//     instructions per tile in the probing loops of the variable windows.)
//   * Rows that need more than the funnel shift — the window starts / ends inside a gap run (patched with flank
//     bases, core:671-682), holds IUPAC cells, runs past a ragged row end, or (tables only) holds a gap and therefore
//     needs the base-5 key — are recorded in a block-private list and handled densely, one per thread, at the end.
#define HIST_THREADS 256
#define WIN_TILES 16
#define WIN_ROWS (HIST_THREADS * WIN_TILES)
#define DEFER_CAP 8000  // deferred (window, row) pairs per block; beyond it rows are handled where they stand

struct RawWin {
    uint32_t a, c, g, t, gapv;
    bool special;  // needs patching / expansion / ragged handling
};
__device__ __forceinline__ RawWin win_cut(const uint4& q0, const uint4& q1, int sh, uint32_t kmask, int p, int k, int len) {
    RawWin r;
    r.a = __funnelshift_r(q0.x, q1.x, sh) & kmask;
    r.c = __funnelshift_r(q0.y, q1.y, sh) & kmask;
    r.g = __funnelshift_r(q0.z, q1.z, sh) & kmask;
    r.t = __funnelshift_r(q0.w, q1.w, sh) & kmask;
    r.gapv = ~(r.a | r.c | r.g | r.t) & kmask;
    r.special = (p + k > len) || ((((r.gapv & 1u) | ((r.gapv >> (k - 1)) & 1u)) != 0u) && r.gapv != kmask) ||
                mpb_multi(r.a, r.c, r.g, r.t) != 0u;
    return r;
}

// the code / key most lanes of the warp share (vote on the first tile that has any)
template <class T>
__device__ __forceinline__ T warp_majority(unsigned mask, bool mine, T val) {
    unsigned peers = 0;
    if (mine) peers = __match_any_sync(mask, val);
    const unsigned cnt = __popc(peers);
    const unsigned mx = __reduce_max_sync(0xffffffffu, cnt);
    const int leader = __ffs(__ballot_sync(0xffffffffu, cnt == mx && mine)) - 1;
    return __shfl_sync(0xffffffffu, val, leader);
}

// host: groups (first batch index, count) of consecutive windows that share their column word
static void mpb_window_groups(const int32_t* win_pos, int nw, std::vector<int2>& groups) {
    groups.clear();
    for (int i = 0; i < nw;) {
        int j = i + 1;
        while (j < nw && j - i < 32 && (win_pos[j] >> 5) == (win_pos[i] >> 5)) ++j;
        groups.push_back(make_int2(i, j - i));
        i = j;
    }
}

// ------------------------------------------------------------------------------------------------------
// entropy prefilter: a lower bound of a window's total entropy from a coarse view of its k-mers
// ------------------------------------------------------------------------------------------------------
// Every item the reference counts for tBit (each expansion of a cover row, each gap row; core:602-614) is mapped to a
// 16-bit code: a hash of the 2-bit bases of ALL its cells (a gap cell, or the lowest base of an IUPAC cell of a gap
// row, counts as that base).  The code is a function of the item's identity, so the bins merge categories, and merging
// can only lower sum(-p log p) (f(a+b) <= f(a)+f(b) for f = -x log x): the entropy of the 65536 bins is a lower bound
// of tBit, and windows whose bound is above the gate never need a table.  Hashing the whole window (instead of
// projecting onto a few cells) keeps the bound tight for windows that are only partly variable: on the synthetic
// workload it lets through exactly the windows the exact gate accepts.
#define PRE_BINS 65536
__device__ __forceinline__ uint32_t pre_code(uint32_t c, uint32_t g, uint32_t t) {
    const uint32_t lo = c | t, hi = g | t;  // bit j of (lo, hi) = base of cell j as 2 bits (A=00 C=01 G=10 T=11)
    return ((lo ^ (hi << 7) ^ (hi >> 9)) * 0x9E3779B1u) >> 16;
}

// one deferred row of the prefilter: a cover row expansion or a gap row, patched window already loaded
__device__ __forceinline__ void pre_row(const Win& w, int v, unsigned int* B, int* err) {
    const bool isgap = __popc(w.gapv) > v;
    if (w.multi == 0 || isgap) {
        uint32_t c = w.c, g = w.g, tt = w.t;
        if (w.multi) {  // gap row holding IUPAC cells: lowest base of every cell
            const uint32_t a = w.a;
            c &= ~a;
            g &= ~(a | c);
            tt &= ~(a | c | g);
        }
        atomicAdd(&B[pre_code(c, g, tt)], 1u);
    } else {
        const uint32_t total = mpb_expansions(w);
        if (total > MPB_MAX_EXP) {
            atomicOr(err, MPB_ERR_EXPAND);
        } else {
            for (uint32_t e = 0; e < total; ++e) {
                uint32_t a, c, g, tt;
                mpb_expand(w, e, a, c, g, tt);
                atomicAdd(&B[pre_code(c, g, tt)], 1u);
            }
        }
    }
}

__global__ void __launch_bounds__(HIST_THREADS)
k_prefilter(const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq, const int32_t* __restrict__ lens, int k, int v,
            const int32_t* __restrict__ win_pos, const int2* __restrict__ groups, int n_groups,
            unsigned int* __restrict__ bins, int* __restrict__ err) {
    __shared__ unsigned int s_defer[DEFER_CAP];
    __shared__ unsigned int s_ndefer;
    __shared__ int s_p[HIST_THREADS / 32][32];            // window start columns of the group, per warp
    __shared__ uint32_t s_major[HIST_THREADS / 32][32];   // majority code of every window of the group, per warp
    const uint32_t kmask = (1u << k) - 1u;
    int lane;
    asm("mov.u32 %0, %%laneid;" : "=r"(lane));
    const int warp = threadIdx.x >> 5;
    const int64_t row_base = (int64_t)blockIdx.x * WIN_ROWS;
    if (threadIdx.x == 0) s_ndefer = 0;
    __syncthreads();
    int gslot = 0;
    for (int g = blockIdx.y; g < n_groups; g += gridDim.y, ++gslot) {
        const int2 gr = groups[g];
        __syncwarp();
        s_p[warp][lane] = lane < gr.y ? win_pos[gr.x + lane] : 0;  // lane j <-> window j of the group
        __syncwarp();
        const uint4* __restrict__ wbase = reinterpret_cast<const uint4*>(pl) + (int64_t)(s_p[warp][0] >> 5) * nsp;
        uint32_t my_major = 0;
        unsigned my_count = 0, have_mask = 0;
        for (int t = 0; t < WIN_TILES; ++t) {
            const int64_t tile0 = row_base + t * HIST_THREADS;
            if (tile0 >= n_seq) break;  // uniform
            const int64_t s = tile0 + threadIdx.x;
            const bool valid = s < n_seq;
            uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
            int len = 0;
            if (valid) {
                q0 = __ldg(wbase + s);
                q1 = __ldg(wbase + nsp + s);
                len = __ldg(lens + s);
            }
#pragma unroll 2
            for (int j = 0; j < gr.y; ++j) {
                const int p = s_p[warp][j];
                unsigned int* B = bins + (long long)(gr.x + j) * PRE_BINS;
                bool plain = false;
                uint32_t code = 0;
                if (valid) {
                    const RawWin r = win_cut(q0, q1, p & 31, kmask, p, k, len);
                    if (r.special) {
                        const unsigned idx = atomicAdd(&s_ndefer, 1u);
                        if (idx < DEFER_CAP) {
                            s_defer[idx] = ((unsigned)(gslot * 32 + j) << 12) | (unsigned)(t * HIST_THREADS + threadIdx.x);
                        } else {  // list full: handle the row here
                            Win w;
                            if (!mpb_load_window(pl, nsp, s, len, p, k, kmask, w)) atomicOr(err, MPB_ERR_SHORT_ROW);
                            pre_row(w, v, B, err);
                        }
                    } else {
                        plain = true;
                        code = pre_code(r.c, r.g, r.t);
                    }
                }
                const unsigned pm = __ballot_sync(0xffffffffu, plain);
                uint32_t major;
                if (!((have_mask >> j) & 1u) && pm) {
                    major = warp_majority<uint32_t>(pm, plain, code);
                    if (lane == j) {
                        my_major = major;
                        s_major[warp][j] = major;
                    }
                    have_mask |= 1u << j;
                    __syncwarp();
                } else {
                    major = s_major[warp][j];
                }
                const unsigned eq = __ballot_sync(0xffffffffu, plain && code == major);
                if (lane == j) my_count += __popc(eq);
                if (plain && code != major) atomicAdd(&B[code], 1u);
            }
        }
        if (lane < gr.y && my_count) atomicAdd(&bins[(long long)(gr.x + lane) * PRE_BINS + my_major], my_count);
    }
    __syncthreads();
    const unsigned nd = s_ndefer < DEFER_CAP ? s_ndefer : DEFER_CAP;
    for (unsigned i = threadIdx.x; i < nd; i += HIST_THREADS) {
        const unsigned e = s_defer[i];
        const unsigned ws = e >> 12;
        const int wi = groups[blockIdx.y + (int)(ws >> 5) * gridDim.y].x + (int)(ws & 31u);
        const int64_t s = row_base + (e & 0xFFFu);
        Win w;
        if (!mpb_load_window(pl, nsp, s, lens[s], win_pos[wi], k, kmask, w)) atomicOr(err, MPB_ERR_SHORT_ROW);
        pre_row(w, v, bins + (long long)wi * PRE_BINS, err);
    }
}

// ------------------------------------------------------------------------------------------------------
// window haplotype tables (core:651-711) + the row classes and patched windows the column scan needs
// ------------------------------------------------------------------------------------------------------
// one deferred row of the table build: patching, gap test, IUPAC expansion in product order, exceptions
__device__ __forceinline__ void hist_row(const uint32_t* __restrict__ pl, int64_t nsp, int64_t s, int len, int p, int k,
                                         int v, uint32_t kmask, long long row0, int wi, uint64_t* K, uint32_t* C,
                                         uint64_t* F, uint32_t* E, int log2cap, unsigned long long* __restrict__ gap_n,
                                         unsigned long long* __restrict__ iupac_gap_n, int32_t* __restrict__ exc,
                                         unsigned long long* __restrict__ exc_n, long long exc_max,
                                         unsigned long long* __restrict__ n_entries, uint32_t* __restrict__ gap_bits,
                                         long long nwords, uint4* __restrict__ spec_win, int32_t* __restrict__ spec_row,
                                         unsigned long long* __restrict__ spec_n, long long spec_cap, int mode,
                                         int* __restrict__ err) {
    // mode 0: plain row already classified where it stood (gap bit, gap count); 1: special row; 2: plain row holding
    // gaps whose gap test is still to do (column-domain pass)
    const uint64_t gs = (uint64_t)(row0 + s);
    Win w;
    if (!mpb_load_window(pl, nsp, s, len, p, k, kmask, w)) atomicOr(err, MPB_ERR_SHORT_ROW);
    const bool isgap = __popc(w.gapv) > v;
    if (mode != 0) {
        if (isgap) {
            atomicAdd(&gap_n[wi], 1ull);
            atomicOr(&gap_bits[(long long)wi * nwords + (s >> 5)], 1u << (s & 31));
        } else if (mode == 1) {  // the patched window itself, for the column scan's special pass
            const unsigned long long slot = atomicAdd(&spec_n[wi], 1ull);
            if ((long long)slot < spec_cap) {
                spec_win[(long long)wi * spec_cap + slot] = make_uint4(w.a, w.c, w.g, w.t);
                spec_row[(long long)wi * spec_cap + slot] = (int32_t)s;
            }
        }
    }
    if (w.multi == 0) {
        mpb_table_add(K, C, F, log2cap, mpb_key(w.c, w.g, w.t, w.gapv, k), 1u, gs << 16, err, &n_entries[wi], E);
    } else if (!isgap) {
        const uint32_t total = mpb_expansions(w);
        if (total > MPB_MAX_EXP) {
            atomicOr(err, MPB_ERR_EXPAND);
        } else {
            for (uint32_t e = 0; e < total; ++e) {
                uint32_t a, c, g, tt;
                mpb_expand(w, e, a, c, g, tt);
                mpb_table_add(K, C, F, log2cap, mpb_key(c, g, tt, w.gapv, k), 1u, (gs << 16) | e, err, &n_entries[wi], E);
            }
        }
    } else {  // gap row holding IUPAC cells: not table material (its raw k-mer needs 4 bits per cell)
        atomicAdd(&iupac_gap_n[wi], 1ull);
        const unsigned long long slot = atomicAdd(exc_n, 1ull);
        if ((long long)slot < exc_max) {
            exc[2 * slot] = wi;
            exc[2 * slot + 1] = (int32_t)s;
        }
    }
}

#define HIST_DEFER_CAP 4000  // deferred special / gapped rows per block
#define HIST_QCAP 256        // queued minority rows per warp

// insert a warp's queued minority rows, one per lane at a time
__device__ __forceinline__ void hist_flush(const unsigned long long* __restrict__ qkey, const unsigned int* __restrict__ qmeta,
                                           unsigned qn, int lane, uint64_t* __restrict__ keys, uint32_t* __restrict__ cnt,
                                           uint64_t* __restrict__ first, uint32_t* __restrict__ elist,
                                           unsigned long long* __restrict__ n_entries, int log2cap, long long row0,
                                           int64_t row_base, int* __restrict__ err) {
    __syncwarp();
    const uint64_t cap = 1ull << log2cap;
    for (unsigned i = lane; i < qn; i += 32) {
        const unsigned m = qmeta[i];
        const unsigned wi = m & 0xFFFFu;
        const uint64_t s = (uint64_t)(row_base + (m >> 16));
        mpb_table_add(keys + (uint64_t)wi * cap, cnt + (uint64_t)wi * cap, first + (uint64_t)wi * cap, log2cap, qkey[i], 1u,
                      (uint64_t)(row0 + s) << 16, err, &n_entries[wi], elist + (uint64_t)wi * cap);
    }
    __syncwarp();
}

__global__ void __launch_bounds__(HIST_THREADS)
k_hist(const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq, const int32_t* __restrict__ lens, int k, int v,
       const int32_t* __restrict__ win_pos, const int2* __restrict__ groups, int n_groups, uint64_t* __restrict__ keys,
       uint32_t* __restrict__ cnt, uint64_t* __restrict__ first, int log2cap, unsigned long long* __restrict__ gap_n,
       unsigned long long* __restrict__ iupac_gap_n, int32_t* __restrict__ exc, unsigned long long* __restrict__ exc_n,
       long long exc_max, long long row0, unsigned long long* __restrict__ n_entries, uint32_t* __restrict__ elist,
       uint32_t* __restrict__ spec_bits, uint32_t* __restrict__ gap_bits, long long nwords, uint4* __restrict__ spec_win,
       int32_t* __restrict__ spec_row, unsigned long long* __restrict__ spec_n, long long spec_cap,
       int* __restrict__ err) {
    __shared__ unsigned int s_defer[HIST_DEFER_CAP];
    __shared__ unsigned int s_ndefer;
    __shared__ int s_p[HIST_THREADS / 32][32];                      // window start columns of the group, per warp
    __shared__ unsigned long long s_major[HIST_THREADS / 32][32];   // majority key of every window of the group, per warp
    // minority rows wait in a per-warp queue and are inserted 32 at a time: a table insert is three dependent trips to
    // L2, and done where the row stands it runs with a few of the 32 lanes
    __shared__ unsigned long long s_qkey[HIST_THREADS / 32][HIST_QCAP];
    __shared__ unsigned int s_qmeta[HIST_THREADS / 32][HIST_QCAP];  // window index | row within the block << 16
    unsigned qn = 0;
    const uint32_t kmask = (1u << k) - 1u;
    const uint64_t cap = 1ull << log2cap;
    int lane;
    asm("mov.u32 %0, %%laneid;" : "=r"(lane));
    const int warp = threadIdx.x >> 5;
    const int64_t row_base = (int64_t)blockIdx.x * WIN_ROWS;
    if (threadIdx.x == 0) s_ndefer = 0;
    __syncthreads();
    int gslot = 0;
    for (int g = blockIdx.y; g < n_groups; g += gridDim.y, ++gslot) {
        const int2 gr = groups[g];
        __syncwarp();
        s_p[warp][lane] = lane < gr.y ? win_pos[gr.x + lane] : 0;  // lane j <-> window j of the group
        __syncwarp();
        const uint4* __restrict__ wbase = reinterpret_cast<const uint4*>(pl) + (int64_t)(s_p[warp][0] >> 5) * nsp;
        unsigned long long my_major = 0, my_first = 0;
        unsigned my_count = 0, my_gaps = 0, have_mask = 0;
        for (int t = 0; t < WIN_TILES; ++t) {
            const int64_t tile0 = row_base + t * HIST_THREADS;
            if (tile0 >= n_seq) break;  // uniform
            const int64_t s = tile0 + threadIdx.x;
            const bool valid = s < n_seq;
            uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
            int len = 0;
            if (valid) {
                q0 = __ldg(wbase + s);
                q1 = __ldg(wbase + nsp + s);
                len = __ldg(lens + s);
            }
            const long long word = tile0 / 32 + warp;
            for (int j = 0; j < gr.y; ++j) {
                const int p = s_p[warp][j];
                const int wi = gr.x + j;
                uint64_t* K = keys + (uint64_t)wi * cap;
                uint32_t* C = cnt + (uint64_t)wi * cap;
                uint64_t* F = first + (uint64_t)wi * cap;
                uint32_t* E = elist + (uint64_t)wi * cap;
                bool plain = false, simple = false, isgap = false, late = false, late_special = false;
                unsigned long long key = 0;
                if (valid) {
                    const RawWin r = win_cut(q0, q1, p & 31, kmask, p, k, len);
                    plain = !r.special;
                    isgap = plain && __popc(r.gapv) > v;
                    simple = plain && r.gapv == 0u;  // gap-free: the 2-bit key; rows holding gaps need the base-5 key
                    if (simple) {
                        key = (unsigned long long)(r.c | r.t) | ((unsigned long long)(r.g | r.t) << k);
                    } else {
                        const unsigned idx = atomicAdd(&s_ndefer, 1u);
                        if (idx < HIST_DEFER_CAP) {
                            s_defer[idx] = ((unsigned)(gslot * 32 + j) << 13) | (r.special ? 0x1000u : 0u) |
                                           (unsigned)(t * HIST_THREADS + threadIdx.x);
                        } else {  // list full: handle the row in this iteration, after the class words are stored
                            late = true;
                            late_special = r.special;
                        }
                    }
                }
                const unsigned pm = __ballot_sync(0xffffffffu, plain);
                const unsigned gb = __ballot_sync(0xffffffffu, plain && isgap);
                if (lane == j) my_gaps += __popc(gb);
                if (lane == 0 && word < nwords) {  // row classes of this 32-sequence word for the column scan
                    spec_bits[(long long)wi * nwords + word] = ~pm;  // (padding rows count as special)
                    gap_bits[(long long)wi * nwords + word] = gb;
                }
                __syncwarp();  // the class words are in place before a late row ORs its gap bit in
                const unsigned sm = __ballot_sync(0xffffffffu, simple);
                unsigned long long major;
                if (!((have_mask >> j) & 1u) && sm) {
                    major = warp_majority<unsigned long long>(sm, simple, key);
                    if (lane == j) {
                        my_major = major;
                        s_major[warp][j] = major;
                    }
                    have_mask |= 1u << j;
                    __syncwarp();
                } else {
                    major = s_major[warp][j];
                }
                const unsigned eq = __ballot_sync(0xffffffffu, simple && key == major);
                if (lane == j) {
                    if (my_count == 0 && eq) my_first = (unsigned long long)(row0 + tile0 + warp * 32 + (__ffs(eq) - 1)) << 16;
                    my_count += __popc(eq);
                }
                {
                    const unsigned mm = __ballot_sync(0xffffffffu, simple && key != major);
                    if (mm) {
                        if (qn + 32 > HIST_QCAP) {  // warp-uniform: make room first
                            hist_flush(s_qkey[warp], s_qmeta[warp], qn, lane, keys, cnt, first, elist, n_entries, log2cap, row0,
                                       row_base, err);
                            qn = 0;
                        }
                        if (simple && key != major) {
                            const unsigned slot = qn + __popc(mm & ((1u << lane) - 1u));
                            s_qkey[warp][slot] = key;
                            s_qmeta[warp][slot] = (unsigned)wi | ((unsigned)(t * HIST_THREADS + threadIdx.x) << 16);
                        }
                        qn += __popc(mm);
                        __syncwarp();
                    }
                }
                if (late)
                    hist_row(pl, nsp, s, len, p, k, v, kmask, row0, wi, K, C, F, E, log2cap, gap_n, iupac_gap_n, exc, exc_n,
                             exc_max, n_entries, gap_bits, nwords, spec_win, spec_row, spec_n, spec_cap, late_special ? 1 : 0, err);
            }
        }
        if (lane < gr.y) {
            const int wi = gr.x + lane;
            if (my_count)
                mpb_table_add(keys + (uint64_t)wi * cap, cnt + (uint64_t)wi * cap, first + (uint64_t)wi * cap, log2cap, my_major,
                              my_count, my_first, err, &n_entries[wi], elist + (uint64_t)wi * cap);
            if (my_gaps) atomicAdd(&gap_n[wi], (unsigned long long)my_gaps);
        }
    }
    hist_flush(s_qkey[warp], s_qmeta[warp], qn, lane, keys, cnt, first, elist, n_entries, log2cap, row0, row_base, err);
    __syncthreads();
    const unsigned nd = s_ndefer < HIST_DEFER_CAP ? s_ndefer : HIST_DEFER_CAP;
    for (unsigned i = threadIdx.x; i < nd; i += HIST_THREADS) {
        const unsigned e = s_defer[i];
        const unsigned ws = e >> 13;
        const int wi = groups[blockIdx.y + (int)(ws >> 5) * gridDim.y].x + (int)(ws & 31u);
        const int64_t s = row_base + (e & 0xFFFu);
        hist_row(pl, nsp, s, lens[s], win_pos[wi], k, v, kmask, row0, wi, keys + (uint64_t)wi * cap, cnt + (uint64_t)wi * cap,
                 first + (uint64_t)wi * cap, elist + (uint64_t)wi * cap, log2cap, gap_n, iupac_gap_n, exc, exc_n, exc_max,
                 n_entries, gap_bits, nwords, spec_win, spec_row, spec_n, spec_cap, (e & 0x1000u) != 0u ? 1 : 0, err);
    }
}

// per window: sum(c) and sum(c log2 c) over the bins
__global__ void __launch_bounds__(256)
k_prefilter_sums(const unsigned int* __restrict__ bins, double* __restrict__ s0, double* __restrict__ s1) {
    const unsigned int* B = bins + (long long)blockIdx.x * PRE_BINS;
    double a0 = 0, a1 = 0;
    for (int i = threadIdx.x; i < PRE_BINS; i += 256) {
        const unsigned int c = B[i];
        if (c) {
            a0 += (double)c;
            if (c > 1) a1 += (double)c * log2((double)c);
        }
    }
    __shared__ double sh0[8], sh1[8];
    for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    if ((threadIdx.x & 31) == 0) {
        sh0[threadIdx.x >> 5] = a0;
        sh1[threadIdx.x >> 5] = a1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) {
            a0 += sh0[w];
            a1 += sh1[w];
        }
        s0[blockIdx.x] = a0;
        s1[blockIdx.x] = a1;
    }
}

// ------------------------------------------------------------------------------------------------------
// column-domain window passes
// ------------------------------------------------------------------------------------------------------
// The row-domain passes above spend ~80 (prefilter) / ~210 (tables) warp instructions per (window, 32 rows) to find out,
// row by row, that most rows of a conserved window carry the same k-mer (both are instruction-issue bound).  On the column
// view (colp: one bit per sequence, 32 sequences per word) that question is an AND: with lane = column and a word of 32
// rows per warp, "row equals the reference k-mer R_w of window w" is the AND over the window's columns of
// plane[column][base R_w has there] — a sliding AND over k lanes, done for all windows that start in the lanes' columns
// by log2(k) shuffles.  The same shuffles give "any gap", "any IUPAC cell", "all gaps" and the two edge cells, i.e. the
// reference's row classes (core:666-687): special rows (edge gap, IUPAC, ragged), gap rows, plain rows.  Per (window,
// 32 rows) that is ~5 instructions; rows equal to R_w and all-gap rows are counted in bulk, and only the others — the
// minority haplotypes, rows holding inner gaps, special rows — are queued (block-shared queue, warp-aggregated) and
// handled on the row view with all lanes busy.  R_w is the per-column frequent base of a row sample (mpb_msa::cons):
// any reference k-mer gives the same tables, a frequent one leaves few rows for the queue.
#define CW_THREADS 256
#define CW_WARPS (CW_THREADS / 32)
#define CW_WPW 16                         // words per warp and block
#define CW_WORDS (CW_WARPS * CW_WPW)
#define CW_ROWS (CW_WORDS * 32)           // 4096 rows per block (12 bits in a queue entry)
#define CW_QCAP 10240
#define CW_QROOM 7680                     // most entries one pass of the block adds: 8 warps x 30 windows x 32 rows

struct ColClass {
    uint32_t plain, agp, match;  // plain rows; plain all-gap rows; gap-free plain rows equal to the reference k-mer
};

// lane = column cs + lane; A..T = that column's plane words of one 32-sequence word; cb = the column's reference base.
// Valid for the windows starting in lanes 0 .. 32 - k.
__device__ __forceinline__ ColClass col_classify(uint32_t A, uint32_t C, uint32_t G, uint32_t T, int cb, int k, int L,
                                                 uint32_t vm, uint32_t ragged) {
    const uint32_t gapc = ~(A | C | G | T);
    uint32_t anygap = gapc, allgap = gapc;
    uint32_t anymul = mpb_multi(A, C, G, T);
    uint32_t alleq = cb == 0 ? A : cb == 1 ? C : cb == 2 ? G : T;
    for (int o = 1; o < L; o <<= 1) {  // windows of L = 2^j <= k columns by doubling
        anygap |= __shfl_down_sync(0xffffffffu, anygap, o);
        anymul |= __shfl_down_sync(0xffffffffu, anymul, o);
        allgap &= __shfl_down_sync(0xffffffffu, allgap, o);
        alleq &= __shfl_down_sync(0xffffffffu, alleq, o);
    }
    const int d = k - L;  // two overlapping windows of L columns cover k
    anygap |= __shfl_down_sync(0xffffffffu, anygap, d);
    anymul |= __shfl_down_sync(0xffffffffu, anymul, d);
    allgap &= __shfl_down_sync(0xffffffffu, allgap, d);
    alleq &= __shfl_down_sync(0xffffffffu, alleq, d);
    const uint32_t last = __shfl_down_sync(0xffffffffu, gapc, k - 1);
    const uint32_t special = (((gapc | last) & ~allgap) | anymul | ragged);
    ColClass r;
    r.plain = ~special & vm;
    r.agp = r.plain & allgap;
    r.match = r.plain & ~anygap & alleq;
    return r;
}

// rows of this word whose sequence ends before the lane's window does (lane's window ends at column `need`)
__device__ __forceinline__ uint32_t col_ragged(const int32_t* __restrict__ lens, int64_t s_lane, int64_t n_seq, int need,
                                               int pend) {
    int len_l = 0x7FFFFFFF;
    if (s_lane < n_seq) len_l = __ldg(lens + s_lane);
    const int minlen = __reduce_min_sync(0xffffffffu, len_l);
    uint32_t ragged = 0;
    if (minlen < pend) {  // uniform; rare
        for (int r = 0; r < 32; ++r) {
            const int lr = __shfl_sync(0xffffffffu, len_l, r);
            ragged |= (lr < need ? 1u : 0u) << r;
        }
    }
    return ragged;
}

// queue the set bits of every lane's word (row = row_in_block0 + bit) as entries wi | row << 16: one shared-memory
// atomic per warp, the lanes write their own runs
__device__ __forceinline__ void cw_push(uint32_t bits, unsigned wi, unsigned row_in_block0, unsigned int* s_q,
                                        unsigned int* s_qn, int lane) {
    const unsigned n = __popc(bits);
    unsigned incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    const unsigned total = __shfl_sync(0xffffffffu, incl, 31);
    if (total == 0) return;  // uniform
    unsigned base = 0;
    if (lane == 31) base = atomicAdd(s_qn, total);
    base = __shfl_sync(0xffffffffu, base, 31) + incl - n;
    while (bits) {
        const unsigned b = __ffs(bits) - 1;
        bits &= bits - 1;
        s_q[base++] = wi | ((row_in_block0 + b) << 16);
    }
}

struct HistOut {
    uint64_t* keys;
    uint32_t* cnt;
    uint64_t* first;
    uint32_t* elist;
    int log2cap;
    unsigned long long *gap_n, *iupac_gap_n, *exc_n, *n_entries, *spec_n;
    int32_t* exc;
    long long exc_max, row0, nwords, spec_cap;
    uint32_t *spec_bits, *gap_bits;
    uint4* spec_win;
    int32_t* spec_row;
};

// make sure first[slot of key] <= ord for a key that is already in the table (a warp-mate has just inserted it)
__device__ __forceinline__ void mpb_table_min_first(const uint64_t* __restrict__ keys, uint64_t* __restrict__ first,
                                                    int log2cap, uint64_t key, uint64_t ord) {
    const uint32_t mask = (1u << log2cap) - 1u;
    const uint32_t last_probe = mask < 8191u ? mask : 8191u;
    uint32_t h = mpb_hash(key, log2cap);
    for (uint32_t probe = 0; probe <= last_probe; ++probe) {
        const uint64_t cur = *((volatile const uint64_t*)&keys[h]);
        if (cur == key) {
            if (*((volatile uint64_t*)&first[h]) > ord) atomicMin((unsigned long long*)&first[h], (unsigned long long)ord);
            return;
        }
        if (cur == MPB_KEY_EMPTY_D) return;  // (cannot happen: the leader's insert is ordered before this probe)
        h = (h + 1) & mask;
    }
}

#define CW_Q2CAP 1024  // rows of one flush that need the general path (gaps, patching, IUPAC expansion)

// the queued rows of the table build, on the row view.  Pass 1, every queued row: cut the window; a gap-free plain row
// is a table insert — rows of one warp that carry the same k-mer of the same window (clade variants, frequent single
// mutants) are inserted once, with their number — the others are set aside.  Pass 2, the rows set aside, with all lanes
// busy again: patching, gap test, expansion, base-5 keys (hist_row).
__device__ __forceinline__ void hist_col_flush(const uint32_t* __restrict__ pl, int64_t nsp, const int32_t* __restrict__ lens,
                                               int k, int v, uint32_t kmask, const int32_t* __restrict__ win_pos,
                                               const HistOut& o, int64_t row_base, const unsigned int* s_q,
                                               unsigned int* s_qn, unsigned int* s_q2, unsigned int* s_q2n,
                                               int short_rows, int* __restrict__ err) {
    __syncthreads();
    const unsigned n = *s_qn;
    const uint64_t cap = 1ull << o.log2cap;
    const int lane = threadIdx.x & 31;
    for (unsigned i0 = 0; i0 < n; i0 += CW_THREADS) {  // whole warps stay together for the votes
        const unsigned i = i0 + threadIdx.x;
        const bool have = i < n;
        int wi = -1;
        int64_t s = 0;
        bool simple = false, special = false;
        unsigned long long key = 0;
        unsigned e = 0;
        if (have) {
            e = s_q[i];
            wi = (int)(e & 0xFFFFu);
            s = row_base + (e >> 16);
            const int p = __ldg(win_pos + wi);
            const uint4* wb = reinterpret_cast<const uint4*>(pl) + (int64_t)(p >> 5) * nsp + s;
            const uint4 q0 = __ldg(wb), q1 = __ldg(wb + nsp);
            const RawWin r = win_cut(q0, q1, p & 31, kmask, p, k, short_rows ? __ldg(lens + s) : 0x7FFFFFFF);
            special = r.special;
            simple = !r.special && r.gapv == 0u;
            key = (unsigned long long)(r.c | r.t) | ((unsigned long long)(r.g | r.t) << k);
        }
        const unsigned sm = __ballot_sync(0xffffffffu, simple);
        if (simple) {
            const unsigned peers = __match_any_sync(sm, key) & __match_any_sync(sm, wi);
            const int leader = __ffs(peers) - 1;
            const uint64_t ord = (uint64_t)(o.row0 + s) << 16;
            if (lane == leader)
                mpb_table_add(o.keys + (uint64_t)wi * cap, o.cnt + (uint64_t)wi * cap, o.first + (uint64_t)wi * cap, o.log2cap,
                              key, (uint32_t)__popc(peers), ord, err, &o.n_entries[wi], o.elist + (uint64_t)wi * cap);
            const uint64_t ord_leader = __shfl_sync(peers, ord, leader);
            __syncwarp(peers);  // the leader's insert is visible to its peers
            if (lane != leader && ord < ord_leader)  // rows are queued nearly in order: rare
                mpb_table_min_first(o.keys + (uint64_t)wi * cap, o.first + (uint64_t)wi * cap, o.log2cap, key, ord);
        } else if (have) {
            const unsigned idx = atomicAdd(s_q2n, 1u);
            if (idx < CW_Q2CAP) {
                s_q2[idx] = e | (special ? 0x10000000u : 0u);
            } else {  // list full: where the row stands
                const int p = __ldg(win_pos + wi);
                hist_row(pl, nsp, s, __ldg(lens + s), p, k, v, kmask, o.row0, wi, o.keys + (uint64_t)wi * cap,
                         o.cnt + (uint64_t)wi * cap, o.first + (uint64_t)wi * cap, o.elist + (uint64_t)wi * cap, o.log2cap,
                         o.gap_n, o.iupac_gap_n, o.exc, o.exc_n, o.exc_max, o.n_entries, o.gap_bits, o.nwords, o.spec_win,
                         o.spec_row, o.spec_n, o.spec_cap, special ? 1 : 2, err);
            }
        }
    }
    __syncthreads();
    const unsigned n2 = *s_q2n < CW_Q2CAP ? *s_q2n : CW_Q2CAP;
    for (unsigned i = threadIdx.x; i < n2; i += CW_THREADS) {
        const unsigned e = s_q2[i];
        const int wi = (int)(e & 0xFFFFu);
        const int64_t s = row_base + ((e >> 16) & 0xFFFu);
        const int p = __ldg(win_pos + wi);
        hist_row(pl, nsp, s, __ldg(lens + s), p, k, v, kmask, o.row0, wi, o.keys + (uint64_t)wi * cap, o.cnt + (uint64_t)wi * cap,
                 o.first + (uint64_t)wi * cap, o.elist + (uint64_t)wi * cap, o.log2cap, o.gap_n, o.iupac_gap_n, o.exc, o.exc_n,
                 o.exc_max, o.n_entries, o.gap_bits, o.nwords, o.spec_win, o.spec_row, o.spec_n, o.spec_cap,
                 (e & 0x10000000u) ? 1 : 2, err);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        *s_qn = 0;
        *s_q2n = 0;
    }
    __syncthreads();
}

// chunks: (first column, largest window end) of a group of windows that start within 33 - k consecutive columns;
// chunk_win[chunk * 32 + lane] = batch index of the window starting at column first + lane, or -1
__global__ void __launch_bounds__(CW_THREADS)
k_hist_col(const uint32_t* __restrict__ colp, int ncols, const uint8_t* __restrict__ cons, const uint32_t* __restrict__ pl,
           int64_t nsp, int64_t n_seq, const int32_t* __restrict__ lens, int k, int v, const int32_t* __restrict__ win_pos,
           const int2* __restrict__ chunks, const int32_t* __restrict__ chunk_win, int n_chunks, HistOut o,
           int short_rows, int* __restrict__ err) {
    __shared__ unsigned int s_q[CW_QCAP];
    __shared__ unsigned int s_q2[CW_Q2CAP];
    __shared__ unsigned int s_qn, s_q2n;
    const uint32_t kmask = (1u << k) - 1u;
    int lane;
    asm("mov.u32 %0, %%laneid;" : "=r"(lane));
    const int warp = threadIdx.x >> 5;
    const int64_t row_base = (int64_t)blockIdx.x * CW_ROWS;
    const long long word_base = (long long)blockIdx.x * CW_WORDS;
    const uint64_t cap = 1ull << o.log2cap;
    int L = 1;
    while (2 * L <= k) L *= 2;
    const bool ag_gap = k > v;  // an all-gap row is a gap row (core:688) unless the variation allows k gaps
    if (threadIdx.x == 0) {
        s_qn = 0;
        s_q2n = 0;
    }
    __syncthreads();
    for (int ch = blockIdx.y; ch < n_chunks; ch += gridDim.y) {
        const int2 cc = chunks[ch];
        const int wi = chunk_win[ch * 32 + lane];
        const bool lane_ok = wi >= 0 && lane + k <= 32;
        const int col = cc.x + lane;
        const bool colok = col < ncols;
        const int cb = colok ? (int)cons[col] : 0;
        const uint32_t lo_w = __ballot_sync(0xffffffffu, cb & 1), hi_w = __ballot_sync(0xffffffffu, cb & 2);
        const uint64_t major = (uint64_t)((lo_w >> lane) & kmask) | ((uint64_t)((hi_w >> lane) & kmask) << k);
        unsigned my_count = 0, ag_count = 0;
        unsigned long long my_first = 0, ag_first = 0;
        for (int it = 0; it < CW_WPW; ++it) {
            __syncthreads();
            if (s_qn > CW_QCAP - CW_QROOM)  // uniform: the counter is read between two barriers
                hist_col_flush(pl, nsp, lens, k, v, kmask, win_pos, o, row_base, s_q, &s_qn, s_q2, &s_q2n, short_rows, err);
            else
                __syncthreads();
            const long long W = word_base + it * CW_WARPS + warp;
            if (W >= o.nwords) continue;  // (the barriers above are passed by every warp)
            const long long left = (long long)n_seq - W * 32;
            const uint32_t vm = left >= 32 ? 0xFFFFFFFFu : left <= 0 ? 0u : ((1u << left) - 1u);
            uint32_t A = 0, C = 0, G = 0, T = 0;
            if (colok && vm) {
                const uint32_t* base = colp + ((long long)col * 4) * o.nwords + W;
                A = __ldg(base);
                C = __ldg(base + o.nwords);
                G = __ldg(base + 2 * o.nwords);
                T = __ldg(base + 3 * o.nwords);
            }
            const uint32_t ragged = (short_rows && vm) ? col_ragged(lens, W * 32 + lane, n_seq, col + k, cc.y) : 0u;
            const ColClass r = col_classify(A, C, G, T, cb, k, L, vm, ragged);
            uint32_t defer = 0;
            if (lane_ok) {
                o.spec_bits[(long long)wi * o.nwords + W] = ~r.plain;
                o.gap_bits[(long long)wi * o.nwords + W] = ag_gap ? r.agp : 0u;
                if (r.match) {
                    if (my_count == 0) my_first = (unsigned long long)(o.row0 + W * 32 + (__ffs(r.match) - 1)) << 16;
                    my_count += __popc(r.match);
                }
                if (r.agp) {
                    if (ag_count == 0) ag_first = (unsigned long long)(o.row0 + W * 32 + (__ffs(r.agp) - 1)) << 16;
                    ag_count += __popc(r.agp);
                }
                defer = vm & ~(r.match | r.agp);
            }
            cw_push(defer, (unsigned)wi, (unsigned)((it * CW_WARPS + warp) * 32), s_q, &s_qn, lane);
        }
        if (lane_ok) {
            uint64_t* K = o.keys + (uint64_t)wi * cap;
            uint32_t* C = o.cnt + (uint64_t)wi * cap;
            uint64_t* F = o.first + (uint64_t)wi * cap;
            uint32_t* E = o.elist + (uint64_t)wi * cap;
            if (my_count) mpb_table_add(K, C, F, o.log2cap, major, my_count, my_first, err, &o.n_entries[wi], E);
            if (ag_count) {
                mpb_table_add(K, C, F, o.log2cap, mpb_key(0u, 0u, 0u, kmask, k), ag_count, ag_first, err, &o.n_entries[wi], E);
                if (ag_gap) atomicAdd(&o.gap_n[wi], (unsigned long long)ag_count);
            }
        }
    }
    hist_col_flush(pl, nsp, lens, k, v, kmask, win_pos, o, row_base, s_q, &s_qn, s_q2, &s_q2n, short_rows, err);
}

// host: chunks of windows for the column-domain passes (windows sorted by start column; a chunk holds the windows that
// start within 33 - k columns of its first one, at most one per column)
static void mpb_window_chunks(const int32_t* win_pos, int nw, int k, std::vector<int2>& chunks, std::vector<int32_t>& chunk_win) {
    std::vector<int32_t> order(nw);
    for (int i = 0; i < nw; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return win_pos[a] < win_pos[b]; });
    chunks.clear();
    chunk_win.clear();
    const int span = 32 - k;  // a window may start in lanes 0 .. span
    std::vector<char> done(nw, 0);
    int n_done = 0;
    size_t from = 0;
    while (n_done < nw) {
        while (done[order[from]]) ++from;
        const int cs = win_pos[order[from]];
        int2 c = make_int2(cs, cs + k);
        const size_t base = chunk_win.size();
        chunk_win.resize(base + 32, -1);
        for (size_t j = from; j < (size_t)nw; ++j) {
            const int32_t w = order[j];
            const int lane = win_pos[w] - cs;
            if (lane > span) break;
            if (done[w] || chunk_win[base + lane] >= 0) continue;  // (a second window at the same column waits)
            chunk_win[base + lane] = w;
            done[w] = 1;
            ++n_done;
            if (win_pos[w] + k > c.y) c.y = win_pos[w] + k;
        }
        chunks.push_back(c);
    }
}

static bool mpb_use_col_passes() {
    const char* e = getenv("MPB_WINPASS");
    return !(e && strcmp(e, "row") == 0);
}

// blocks along y (window stride) for a window pass: fill whole waves of resident blocks, a few waves deep
template <class Kern>
static unsigned window_pass_gy(mpb_ctx* ctx, Kern kern, unsigned gx, int nw) {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, HIST_THREADS, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
    const long long resident = (long long)per_sm * ctx->sm_count;
    if ((long long)gx * nw <= 16 * resident) return (unsigned)nw;  // one group per block: uniform work, many waves
    long long lo = (resident + gx - 1) / gx, hi = (4 * resident + gx - 1) / gx + 1;
    if (lo < 1) lo = 1;
    if (hi > nw) hi = nw;
    if (lo > hi) lo = hi;
    unsigned best = (unsigned)lo;
    double best_eff = -1;
    for (long long gy = lo; gy <= hi; ++gy) {
        const long long blocks = (long long)gx * gy, waves = (blocks + resident - 1) / resident;
        const double eff = (double)blocks / (double)(waves * resident);
        if (eff >= best_eff) {
            best_eff = eff;
            best = (unsigned)gy;
        }
    }
    return best;
}

extern "C" int mpb_window_prefilter(mpb_msa* m, int k, int v, const int32_t* win_pos, int32_t nw, double* s0_hd,
                                    double* s1_hd) {
    if (!m || !win_pos || !s0_hd || !s1_hd) return fail(MPB_EINVAL, "NULL argument");
    if (k < 8 || k > MPB_MAX_K || v < 0 || nw < 1) return fail(MPB_EINVAL, "prefilter needs 8 <= k <= %d", MPB_MAX_K);
    for (int i = 0; i < nw; ++i)
        if (win_pos[i] < 0 || win_pos[i] >= m->n_col)
            return fail(MPB_EINVAL, "win_pos[%d]=%d outside the alignment", i, win_pos[i]);
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    bool inside = true;  // the bit-sliced kernel walks columns win_pos .. win_pos + k - 1 of the column view
    for (int i = 0; i < nw; ++i) inside = inside && win_pos[i] + k <= m->n_col;
    if (mpb_use_col_passes() && inside && !m->short_rows) return mpb_prefilter_bs(m, k, v, win_pos, nw, s0_hd, s1_hd);
    unsigned int* bins = nullptr;
    CK(cudaMallocAsync(&bins, (size_t)nw * PRE_BINS * 4, ctx->stream));
    CK(cudaMemsetAsync(bins, 0, (size_t)nw * PRE_BINS * 4, ctx->stream));
    InBuf wp(ctx, win_pos, (size_t)nw * 4);
    OutBuf o0(ctx, s0_hd, (size_t)nw * 8), o1(ctx, s1_hd, (size_t)nw * 8);
    if (wp.rc || o0.rc || o1.rc) return MPB_ECUDA;
    {
        const unsigned gx = (unsigned)((m->n_seq + (long long)WIN_ROWS - 1) / (long long)WIN_ROWS);
        std::vector<int2> groups;
        mpb_window_groups(win_pos, nw, groups);
        InBuf gr(ctx, groups.data(), groups.size() * sizeof(int2));
        if (gr.rc) return gr.rc;
        const unsigned gy = window_pass_gy(ctx, k_prefilter, gx, (int)groups.size());
        ctx->pending_units = (double)nw * (double)m->n_seq;
        LAUNCH(ctx, k_prefilter, dim3(gx, gy), HIST_THREADS, 0, m->planes, m->nsp, m->n_seq, m->lens, k, v, wp.dev<int32_t>(),
               gr.dev<int2>(), (int)groups.size(), bins, m->err);
    }
    LAUNCH(ctx, k_prefilter_sums, (unsigned)nw, 256, 0, bins, o0.dev<double>(), o1.dev<double>());
    CK(o0.finish());
    CK(o1.finish());
    CK(cudaFreeAsync(bins, ctx->stream));
    return mpb_check_flags(ctx, m->err);
}

static int hist_alloc_spec(mpb_hist* h, int64_t spec_cap) {
    mpb_ctx* ctx = h->msa->ctx;
    h->spec_cap = spec_cap;
    cudaError_t e = cudaMallocAsync(&h->spec_win, (size_t)h->nw * spec_cap * sizeof(uint4), ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->spec_row, (size_t)h->nw * spec_cap * 4, ctx->stream);
    if (e != cudaSuccess) return fail(MPB_ENOMEM, "special-row lists (%d windows x %lld rows): %s", h->nw, (long long)spec_cap,
                                      cudaGetErrorString(e));
    return 0;
}

static int hist_launch_build(mpb_hist* h) {
    mpb_msa* m = h->msa;
    mpb_ctx* ctx = m->ctx;
    const int nw = h->nw;
    const uint64_t slots = (uint64_t)nw << h->log2cap;
    CK(cudaMemsetAsync(h->keys, 0xFF, slots * 8, ctx->stream));
    CK(cudaMemsetAsync(h->cnt, 0, slots * 4, ctx->stream));
    CK(cudaMemsetAsync(h->first, 0xFF, slots * 8, ctx->stream));
    CK(cudaMemsetAsync(h->gap_n, 0, (size_t)nw * 8, ctx->stream));
    CK(cudaMemsetAsync(h->iupac_gap_n, 0, (size_t)nw * 8, ctx->stream));
    CK(cudaMemsetAsync(h->n_entries, 0, (size_t)nw * 8, ctx->stream));
    CK(cudaMemsetAsync(h->spec_n, 0, (size_t)nw * 8, ctx->stream));
    CK(cudaMemsetAsync(h->exc_n, 0, 8, ctx->stream));
    if (mpb_use_col_passes()) {
        // A window that runs past the last column takes the reference's left extension (core:683-687) on every row.
        // The column view reads the missing cells as gaps, so such a batch flags its rows like those of a ragged input
        // (lens = n_col): col_ragged marks the rows of those windows special, and hist_row cuts them.
        bool ragged = m->short_rows;
        for (int i = 0; i < nw; ++i) ragged = ragged || h->h_win_pos[i] + h->k > m->n_col;
        std::vector<int2> chunks;
        std::vector<int32_t> chunk_win;
        mpb_window_chunks(h->h_win_pos.data(), nw, h->k, chunks, chunk_win);
        InBuf cd(ctx, chunks.data(), chunks.size() * sizeof(int2)), cw(ctx, chunk_win.data(), chunk_win.size() * 4);
        if (cd.rc || cw.rc) return MPB_ECUDA;
        HistOut o;
        o.keys = h->keys;
        o.cnt = h->cnt;
        o.first = h->first;
        o.elist = h->elist;
        o.log2cap = h->log2cap;
        o.gap_n = h->gap_n;
        o.iupac_gap_n = h->iupac_gap_n;
        o.exc_n = h->exc_n;
        o.n_entries = h->n_entries;
        o.spec_n = h->spec_n;
        o.exc = h->exc;
        o.exc_max = (long long)h->exc_max;
        o.row0 = (long long)m->row0;
        o.nwords = (long long)m->nwords;
        o.spec_cap = (long long)h->spec_cap;
        o.spec_bits = h->spec_bits;
        o.gap_bits = h->gap_bits;
        o.spec_win = h->spec_win;
        o.spec_row = h->spec_row;
        const unsigned gx = (unsigned)((m->nwords + CW_WORDS - 1) / CW_WORDS);
        ctx->pending_units = (double)nw * (double)m->n_seq;
        MPB_LAUNCH_NAMED(ctx, "k_hist", k_hist_col, dim3(gx, (unsigned)chunks.size()), CW_THREADS, 0, m->colp, (m->ncw - 1) * 32,
                         m->cons, m->planes, m->nsp, m->n_seq, m->lens, h->k, h->v, h->win_pos, cd.dev<int2>(),
                         cw.dev<int32_t>(), (int)chunks.size(), o, ragged ? 1 : 0, m->err);
        return 0;
    }
    const unsigned gx = (unsigned)((m->n_seq + (long long)WIN_ROWS - 1) / (long long)WIN_ROWS);
    std::vector<int2> groups;
    mpb_window_groups(h->h_win_pos.data(), nw, groups);
    InBuf gr(ctx, groups.data(), groups.size() * sizeof(int2));
    if (gr.rc) return gr.rc;
    const unsigned gy = window_pass_gy(ctx, k_hist, gx, (int)groups.size());
    ctx->pending_units = (double)nw * (double)m->n_seq;  // (window, sequence) k-mers extracted
    LAUNCH(ctx, k_hist, dim3(gx, gy), HIST_THREADS, 0, m->planes, m->nsp, m->n_seq, m->lens, h->k, h->v, h->win_pos,
           gr.dev<int2>(), (int)groups.size(), h->keys, h->cnt, h->first, h->log2cap, h->gap_n, h->iupac_gap_n, h->exc, h->exc_n, (long long)h->exc_max,
           (long long)m->row0, h->n_entries, h->elist, h->spec_bits, h->gap_bits, (long long)m->nwords, h->spec_win,
           h->spec_row, h->spec_n, (long long)h->spec_cap, m->err);
    return 0;
}

// Allocate the tables of nw windows without filling them from the alignment (owner tables of a sequence-sharded run
// receive their entries through mpb_hist_merge only) when `fill` is 0.
static int hist_create(mpb_msa* m, int k, int v, const int32_t* win_pos, int32_t nw, int log2_cap, int fill, mpb_hist** out) {
    if (!m || !win_pos || !out) return fail(MPB_EINVAL, "NULL argument");
    if (k < 3 || k > MPB_MAX_K) return fail(MPB_EINVAL, "primer length %d outside 3..%d", k, MPB_MAX_K);
    if (v < 0 || nw < 1 || nw > 65535) return fail(MPB_EINVAL, "bad v=%d or nw=%d (at most 65535 windows per batch)", v, nw);
    for (int i = 0; i < nw; ++i)
        if (win_pos[i] < 0 || win_pos[i] >= m->n_col)
            return fail(MPB_EINVAL, "win_pos[%d]=%d outside the alignment", i, win_pos[i]);
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    if (log2_cap <= 0) {
        log2_cap = 6;
        while ((1ll << log2_cap) < 2 * m->n_seq + 64) ++log2_cap;
    }
    if (log2_cap > 31) return fail(MPB_EINVAL, "log2_cap %d too large", log2_cap);
    mpb_hist* h = new mpb_hist();
    h->msa = m;
    h->k = k;
    h->v = v;
    h->nw = nw;
    h->log2cap = log2_cap;
    h->exc_max = 1 << 20;
    h->h_win_pos.assign(win_pos, win_pos + nw);
    const uint64_t slots = (uint64_t)nw << log2_cap;
    cudaError_t e = cudaMallocAsync(&h->keys, slots * 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->cnt, slots * 4, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->first, slots * 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->elist, slots * 4, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->win_pos, (size_t)nw * 4, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->gap_n, (size_t)nw * 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->iupac_gap_n, (size_t)nw * 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->n_entries, (size_t)nw * 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->spec_n, (size_t)nw * 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->exc, (size_t)h->exc_max * 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->exc_n, 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->spec_bits, (size_t)nw * m->nwords * 4, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->gap_bits, (size_t)nw * m->nwords * 4, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->freq, (size_t)nw * 4 * k * 8, ctx->stream);
    if (e == cudaSuccess) e = cudaMallocAsync(&h->nn, (size_t)nw * (k - 1) * 16 * 8, ctx->stream);
    if (e != cudaSuccess) {
        mpb_hist_free(h);
        return fail(MPB_ENOMEM, "haplotype tables (%d windows x 2^%d slots): %s", nw, log2_cap, cudaGetErrorString(e));
    }
    CK(cudaMemcpyAsync(h->win_pos, h->h_win_pos.data(), (size_t)nw * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (!fill) {
        const uint64_t sl = (uint64_t)nw << log2_cap;
        CK(cudaMemsetAsync(h->keys, 0xFF, sl * 8, ctx->stream));
        CK(cudaMemsetAsync(h->cnt, 0, sl * 4, ctx->stream));
        CK(cudaMemsetAsync(h->first, 0xFF, sl * 8, ctx->stream));
        CK(cudaMemsetAsync(h->gap_n, 0, (size_t)nw * 8, ctx->stream));
        CK(cudaMemsetAsync(h->iupac_gap_n, 0, (size_t)nw * 8, ctx->stream));
        CK(cudaMemsetAsync(h->n_entries, 0, (size_t)nw * 8, ctx->stream));
        CK(cudaMemsetAsync(h->spec_n, 0, (size_t)nw * 8, ctx->stream));
        CK(cudaMemsetAsync(h->exc_n, 0, 8, ctx->stream));
        *out = h;
        return 0;
    }
    // special-row lists: room for 1/32 of the rows per window at first; a window with more (gap-rich alignments)
    // reports its true count and the build is repeated once with exactly the room it needs
    int64_t cap = m->n_seq / 32;
    if (cap < 1024) cap = m->n_seq < 1024 ? m->n_seq : 1024;
    for (int attempt = 0; attempt < 2; ++attempt) {
        int rc = hist_alloc_spec(h, cap);
        if (rc == 0) rc = hist_launch_build(h);
        if (rc == 0) rc = mpb_check_flags(ctx, m->err);
        if (rc) {
            mpb_hist_free(h);
            return rc;
        }
        std::vector<unsigned long long> sn(nw);
        CK(cudaMemcpyAsync(sn.data(), h->spec_n, (size_t)nw * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        unsigned long long mx = 0;
        for (auto x : sn) mx = x > mx ? x : mx;
        if ((int64_t)mx <= cap) break;
        if (attempt == 1) {
            mpb_hist_free(h);
            return fail(MPB_EOVERFLOW, "special-row list overflow after resize");
        }
        cudaFreeAsync(h->spec_win, ctx->stream);
        cudaFreeAsync(h->spec_row, ctx->stream);
        h->spec_win = nullptr;
        h->spec_row = nullptr;
        cap = (int64_t)mx;
    }
    *out = h;
    return 0;
}

extern "C" int mpb_hist_build(mpb_msa* m, int k, int v, const int32_t* win_pos, int32_t nw, int log2_cap,
                              mpb_hist** out) {
    return hist_create(m, k, v, win_pos, nw, log2_cap, 1, out);
}

extern "C" int mpb_hist_create_empty(mpb_msa* m, int k, int v, const int32_t* win_pos, int32_t nw, int log2_cap,
                                     mpb_hist** out) {
    return hist_create(m, k, v, win_pos, nw, log2_cap, 0, out);
}

// counters kept by k_hist (host arrays of nw, any may be NULL): gap rows, gap rows holding IUPAC cells, distinct entries
extern "C" int mpb_hist_counts(mpb_hist* h, int64_t* gap_n, int64_t* n_iupac_gap, int64_t* n_entries) {
    if (!h) return fail(MPB_EINVAL, "NULL argument");
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    const size_t bytes = (size_t)h->nw * 8;
    if (gap_n) CK(cudaMemcpyAsync(gap_n, h->gap_n, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (n_iupac_gap) CK(cudaMemcpyAsync(n_iupac_gap, h->iupac_gap_n, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (n_entries) CK(cudaMemcpyAsync(n_entries, h->n_entries, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" void mpb_hist_free(mpb_hist* h) {
    if (!h) return;
    cudaStream_t st = h->msa->ctx->stream;
    void* ptrs[] = {h->keys, h->cnt, h->first, h->elist, h->win_pos, h->gap_n, h->iupac_gap_n, h->n_entries, h->exc,
                    h->exc_n, h->spec_bits, h->gap_bits, h->spec_win, h->spec_row, h->spec_n, h->freq, h->nn};
    for (void* p : ptrs)
        if (p) cudaFreeAsync(p, st);
    delete h;
}

// copy the entries of the selected windows into one compact array: window sel_idx[y]'s entries land at start[y] + (their
// position in the entry list); room for room[y] of them
__global__ void k_hist_export(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ cnt,
                              const uint64_t* __restrict__ first, const uint32_t* __restrict__ elist,
                              const unsigned long long* __restrict__ n_entries, int log2cap,
                              const int32_t* __restrict__ sel_idx, const long long* __restrict__ start,
                              const long long* __restrict__ room, uint64_t* __restrict__ ok, uint32_t* __restrict__ oc,
                              uint64_t* __restrict__ of) {
    const int wi = sel_idx[blockIdx.y];
    const uint64_t cap = 1ull << log2cap;
    const uint64_t base = (uint64_t)wi * cap;
    long long n = (long long)n_entries[wi];
    if (n > room[blockIdx.y]) n = room[blockIdx.y];
    const long long o = start[blockIdx.y];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const uint64_t slot = base + elist[base + i];
        ok[o + i] = keys[slot];
        oc[o + i] = cnt[slot];
        of[o + i] = first[slot];
    }
}

// windows sel_idx[0..n_sel) (host) in THIS order: entries of window sel_idx[i] go to [start[i], start[i] + room[i])
extern "C" int mpb_hist_export_at(mpb_hist* h, int32_t n_sel, const int32_t* sel_idx, const int64_t* start,
                                  const int64_t* room, int64_t total, uint64_t* keys_hd, uint32_t* cnt_hd,
                                  uint64_t* first_hd) {
    if (!h || !sel_idx || !start || !room || !keys_hd || !cnt_hd || !first_hd) return fail(MPB_EINVAL, "NULL argument");
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    for (int i = 0; i < n_sel; ++i)
        if (sel_idx[i] < 0 || sel_idx[i] >= h->nw || start[i] < 0 || room[i] < 0 || start[i] + room[i] > total)
            return fail(MPB_EINVAL, "bad placement of window %d", i);
    if (n_sel < 1 || total <= 0) return 0;
    InBuf si(ctx, sel_idx, (size_t)n_sel * 4), st(ctx, start, (size_t)n_sel * 8), rm(ctx, room, (size_t)n_sel * 8);
    OutBuf ok(ctx, keys_hd, total * 8), oc(ctx, cnt_hd, total * 4), of(ctx, first_hd, total * 8);
    if (si.rc || st.rc || rm.rc || ok.rc || oc.rc || of.rc) return MPB_ECUDA;
    LAUNCH(ctx, k_hist_export, dim3(32, (unsigned)n_sel), 256, 0, h->keys, h->cnt, h->first, h->elist, h->n_entries,
           h->log2cap, si.dev<int32_t>(), st.dev<long long>(), rm.dev<long long>(), ok.dev<uint64_t>(), oc.dev<uint32_t>(),
           of.dev<uint64_t>());
    CK(ok.finish());
    CK(oc.finish());
    CK(of.finish());
    if (ok.is_host() || oc.is_host() || of.is_host()) CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int mpb_hist_export(mpb_hist* h, const uint8_t* sel, const int64_t* win_off, uint64_t* keys_hd,
                               uint32_t* cnt_hd, uint64_t* first_hd) {
    if (!h || !sel || !win_off || !keys_hd || !cnt_hd || !first_hd) return fail(MPB_EINVAL, "NULL argument");
    std::vector<int32_t> idx;
    std::vector<int64_t> start, room;
    for (int i = 0; i < h->nw; ++i) {
        if (sel[i]) {
            idx.push_back(i);
            start.push_back(win_off[i]);
            room.push_back(win_off[i + 1] - win_off[i]);
        } else if (win_off[i + 1] != win_off[i]) {
            return fail(MPB_EINVAL, "win_off reserves room for unselected window %d", i);
        }
    }
    if (idx.empty()) return 0;
    int rc = mpb_hist_export_at(h, (int32_t)idx.size(), idx.data(), start.data(), room.data(), win_off[h->nw], keys_hd,
                                cnt_hd, first_hd);
    if (rc) return rc;
    CK(cudaStreamSynchronize(h->msa->ctx->stream));
    return 0;
}

// entries arrive in n_seg segments (seg_off[n_seg + 1]); segment s belongs to window s % nw (a sharded run receives
// one run of segments per source rank)
__global__ void k_hist_merge(const long long* __restrict__ seg_off, int n_seg, int nw, const uint64_t* __restrict__ in_keys,
                             const uint32_t* __restrict__ in_cnt, const uint64_t* __restrict__ in_first,
                             uint64_t* __restrict__ keys, uint32_t* __restrict__ cnt, uint64_t* __restrict__ first,
                             uint32_t* __restrict__ elist, unsigned long long* __restrict__ n_entries, int log2cap,
                             int* __restrict__ err) {
    const long long total = seg_off[n_seg];
    const uint64_t cap = 1ull << log2cap;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = n_seg;  // largest s with seg_off[s] <= i
        while (hi - lo > 1) {
            int mid = (lo + hi) >> 1;
            if (seg_off[mid] <= i) lo = mid;
            else hi = mid;
        }
        const int w = lo % nw;
        mpb_table_add(keys + (uint64_t)w * cap, cnt + (uint64_t)w * cap, first + (uint64_t)w * cap, log2cap, in_keys[i],
                      in_cnt[i], in_first[i], err, &n_entries[w], elist + (uint64_t)w * cap);
    }
}

extern "C" int mpb_hist_merge_segments(mpb_hist* h, int32_t n_seg, const int64_t* seg_off, const uint64_t* keys_hd,
                                       const uint32_t* cnt_hd, const uint64_t* first_hd) {
    if (!h || !seg_off || !keys_hd || !cnt_hd || !first_hd) return fail(MPB_EINVAL, "NULL argument");
    if (n_seg < 1 || n_seg % h->nw != 0) return fail(MPB_EINVAL, "n_seg must be a multiple of the window count");
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    const int64_t total = seg_off[n_seg];
    if (total <= 0) return 0;
    InBuf off(ctx, seg_off, (size_t)(n_seg + 1) * 8), ik(ctx, keys_hd, total * 8), ic(ctx, cnt_hd, total * 4),
        ifr(ctx, first_hd, total * 8);
    if (off.rc || ik.rc || ic.rc || ifr.rc) return MPB_ECUDA;
    unsigned grid = (unsigned)((total + 255) / 256);
    if (grid > (unsigned)ctx->sm_count * 16) grid = ctx->sm_count * 16;
    LAUNCH(ctx, k_hist_merge, grid, 256, 0, off.dev<long long>(), (int)n_seg, h->nw, ik.dev<uint64_t>(), ic.dev<uint32_t>(),
           ifr.dev<uint64_t>(), h->keys, h->cnt, h->first, h->elist, h->n_entries, h->log2cap, h->msa->err);
    h->have_summary = false;
    return mpb_check_flags(ctx, h->msa->err);
}

extern "C" int mpb_hist_merge(mpb_hist* h, const int64_t* win_off, const uint64_t* keys_hd, const uint32_t* cnt_hd,
                              const uint64_t* first_hd) {
    if (!h) return fail(MPB_EINVAL, "NULL argument");
    return mpb_hist_merge_segments(h, h->nw, win_off, keys_hd, cnt_hd, first_hd);
}

// sharded runs: add foreign gap-row counters to the owner's (they are not table entries)
extern "C" int mpb_hist_add_counts(mpb_hist* h, const int64_t* gap_n, const int64_t* n_iupac_gap) {
    if (!h || !gap_n || !n_iupac_gap) return fail(MPB_EINVAL, "NULL argument");
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(h->gap_n, gap_n, (size_t)h->nw * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(h->iupac_gap_n, n_iupac_gap, (size_t)h->nw * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// One pass over the ENTRY LIST of every window (not over the slots): entropy ingredients, distinct counts, the most
// frequent gap-free haplotype (core:595-600), base counts per column and dinucleotide counts per junction weighted by
// the haplotype counts (core:541-577 restated over the table instead of over a pandas frame of expansion rows).
// SUM_SB blocks share a window; each writes one partial record (combined in fixed order on the host) and adds its
// integer tensors with atomics.
// ------------------------------------------------------------------------------------------------------
#define SUM_THREADS 256
#define SUM_SB 8
struct Best {
    unsigned long long cnt, first, key;
};
__device__ __host__ __forceinline__ bool better(const Best& x, const Best& y) {  // x beats y
    return x.cnt > y.cnt || (x.cnt == y.cnt && x.first < y.first);
}
struct StatsPart {
    double s0c, s1c, s0g, s1g;
    long long nc, ng, ngf;
    Best best;
};

template <bool STATS, bool TENS>
__global__ void __launch_bounds__(SUM_THREADS)
k_hist_summary(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ cnt, const uint64_t* __restrict__ first,
               const uint32_t* __restrict__ elist, const unsigned long long* __restrict__ n_entries, int log2cap, int k,
               int v, const int32_t* __restrict__ sel_idx, StatsPart* __restrict__ part,
               unsigned long long* __restrict__ freq, unsigned long long* __restrict__ nn) {
    // block-private 32-bit counters (native shared-memory atomics; 64-bit ones are CAS loops): a block sees an eighth of
    // a window's entries, whose counts sum to far less than 2^32
    __shared__ unsigned int s_freq[4 * MPB_MAX_K];
    __shared__ unsigned int s_nn[(MPB_MAX_K - 1) * 16];
    const int wi = sel_idx ? sel_idx[blockIdx.y] : blockIdx.y;
    const uint64_t cap = 1ull << log2cap;
    const uint64_t base = (uint64_t)wi * cap;
    const uint32_t kmask = (1u << k) - 1u;
    const long long n = (long long)n_entries[wi];
    for (int i = threadIdx.x; i < 4 * k; i += SUM_THREADS) s_freq[i] = 0;
    for (int i = threadIdx.x; i < (k - 1) * 16; i += SUM_THREADS) s_nn[i] = 0;
    __syncthreads();
    double s0c = 0, s1c = 0, s0g = 0, s1g = 0;
    long long nc = 0, ng = 0, ngf = 0;
    Best best = {0ull, ~0ull, MPB_KEY_EMPTY_D};
    for (long long i = (long long)blockIdx.x * SUM_THREADS + threadIdx.x; i < n; i += (long long)SUM_SB * SUM_THREADS) {
        const uint64_t slot = base + elist[base + i];
        const uint64_t key = keys[slot];
        const uint32_t ci = cnt[slot];
        const double c = (double)ci;
        uint32_t pa, pc, pg, pt, gapv;
        mpb_key_planes(key, k, kmask, pa, pc, pg, pt, gapv);
        const bool is_cover = __popc(gapv) <= v;
        if (STATS && key < MPB_KEY_BASE5_D) {
            ++ngf;
            Best b = {(unsigned long long)ci, first[slot], key};
            if (better(b, best)) best = b;
        }
        const double clog = (!STATS || ci == 1u) ? 0.0 : c * log2(c);  // singletons (most of a variable window) cost no log
        if (is_cover) {
            s0c += c;
            s1c += clog;
            ++nc;
            int prev = -1;
            if (TENS)
            for (int j = 0; j < k; ++j) {
                const int d = ((gapv >> j) & 1u) ? -1 : (int)(((pc >> j) & 1u) + 2u * ((pg >> j) & 1u) + 3u * ((pt >> j) & 1u));
                if (d >= 0) atomicAdd(&s_freq[d * k + j], ci);
                if (j > 0 && d >= 0 && prev >= 0) atomicAdd(&s_nn[(j - 1) * 16 + prev * 4 + d], ci);
                prev = d;
            }
        } else {
            s0g += c;
            s1g += clog;
            ++ng;
        }
    }
    __shared__ double sd[4][SUM_THREADS / 32];
    __shared__ long long sl[3][SUM_THREADS / 32];
    __shared__ Best sbest[SUM_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (STATS)
    for (int o = 16; o > 0; o >>= 1) {
        s0c += __shfl_xor_sync(0xffffffffu, s0c, o);
        s1c += __shfl_xor_sync(0xffffffffu, s1c, o);
        s0g += __shfl_xor_sync(0xffffffffu, s0g, o);
        s1g += __shfl_xor_sync(0xffffffffu, s1g, o);
        nc += __shfl_xor_sync(0xffffffffu, nc, o);
        ng += __shfl_xor_sync(0xffffffffu, ng, o);
        ngf += __shfl_xor_sync(0xffffffffu, ngf, o);
        Best ob;
        ob.cnt = __shfl_xor_sync(0xffffffffu, best.cnt, o);
        ob.first = __shfl_xor_sync(0xffffffffu, best.first, o);
        ob.key = __shfl_xor_sync(0xffffffffu, best.key, o);
        if (better(ob, best)) best = ob;
    }
    if (STATS && lane == 0) {
        sd[0][warp] = s0c;
        sd[1][warp] = s1c;
        sd[2][warp] = s0g;
        sd[3][warp] = s1g;
        sl[0][warp] = nc;
        sl[1][warp] = ng;
        sl[2][warp] = ngf;
        sbest[warp] = best;
    }
    __syncthreads();
    if (STATS && threadIdx.x == 0) {
        StatsPart r = {sd[0][0], sd[1][0], sd[2][0], sd[3][0], sl[0][0], sl[1][0], sl[2][0], sbest[0]};
        for (int w = 1; w < SUM_THREADS / 32; ++w) {
            r.s0c += sd[0][w];
            r.s1c += sd[1][w];
            r.s0g += sd[2][w];
            r.s1g += sd[3][w];
            r.nc += sl[0][w];
            r.ng += sl[1][w];
            r.ngf += sl[2][w];
            if (better(sbest[w], r.best)) r.best = sbest[w];
        }
        part[(long long)wi * SUM_SB + blockIdx.x] = r;
    }
    if (TENS) {
        for (int i = threadIdx.x; i < 4 * k; i += SUM_THREADS)
            if (s_freq[i]) atomicAdd(&freq[(long long)wi * 4 * k + i], (unsigned long long)s_freq[i]);
        for (int i = threadIdx.x; i < (k - 1) * 16; i += SUM_THREADS)
            if (s_nn[i]) atomicAdd(&nn[(long long)wi * (k - 1) * 16 + i], (unsigned long long)s_nn[i]);
    }
}

// all outputs host arrays (any may be NULL); freq / nn also stay on the device for the walk (mpb_walk_dev.cu)
extern "C" int mpb_hist_summary(mpb_hist* h, int64_t* gap_n, double* ent, int64_t* nuniq, uint64_t* mm_key,
                                int64_t* mm_cnt, uint64_t* mm_first, int64_t* n_iupac_gap, int64_t* freq, int64_t* nn) {
    if (!h) return fail(MPB_EINVAL, "NULL argument");
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    const size_t nw = h->nw;
    const int k = h->k;
    const size_t fb = nw * 4 * k * 8, nb = nw * (k - 1) * 16 * 8;
    StatsPart* dpart = nullptr;
    CK(cudaMallocAsync(&dpart, nw * SUM_SB * sizeof(StatsPart), ctx->stream));
    const bool tens = freq != nullptr || nn != nullptr;
    if (tens) {
        CK(cudaMemsetAsync(h->freq, 0, fb, ctx->stream));
        CK(cudaMemsetAsync(h->nn, 0, nb, ctx->stream));
        MPB_LAUNCH_NAMED(ctx, "k_hist_summary", (k_hist_summary<true, true>), dim3(SUM_SB, (unsigned)nw), SUM_THREADS, 0, h->keys,
                         h->cnt, h->first, h->elist, h->n_entries, h->log2cap, k, h->v, (const int32_t*)nullptr, dpart, h->freq,
                         h->nn);
    } else {
        MPB_LAUNCH_NAMED(ctx, "k_hist_summary", (k_hist_summary<true, false>), dim3(SUM_SB, (unsigned)nw), SUM_THREADS, 0, h->keys,
                         h->cnt, h->first, h->elist, h->n_entries, h->log2cap, k, h->v, (const int32_t*)nullptr, dpart, h->freq,
                         h->nn);
    }
    std::vector<StatsPart> part(nw * SUM_SB);
    CK(cudaMemcpyAsync(part.data(), dpart, nw * SUM_SB * sizeof(StatsPart), cudaMemcpyDeviceToHost, ctx->stream));
    std::vector<long long> hg(nw), hi(nw);
    CK(cudaMemcpyAsync(hg.data(), h->gap_n, nw * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(hi.data(), h->iupac_gap_n, nw * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (freq) CK(cudaMemcpyAsync(freq, h->freq, fb, cudaMemcpyDeviceToHost, ctx->stream));
    if (nn) CK(cudaMemcpyAsync(nn, h->nn, nb, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaFreeAsync(dpart, ctx->stream));
    h->have_summary = tens;
    for (size_t w = 0; w < nw; ++w) {
        StatsPart r = part[w * SUM_SB];
        for (int b = 1; b < SUM_SB; ++b) {
            const StatsPart& q = part[w * SUM_SB + b];
            r.s0c += q.s0c;
            r.s1c += q.s1c;
            r.s0g += q.s0g;
            r.s1g += q.s1g;
            r.nc += q.nc;
            r.ng += q.ng;
            r.ngf += q.ngf;
            if (better(q.best, r.best)) r.best = q.best;
        }
        if (gap_n) gap_n[w] = hg[w];
        if (n_iupac_gap) n_iupac_gap[w] = hi[w];
        if (ent) {
            ent[w * 4 + 0] = r.s0c;
            ent[w * 4 + 1] = r.s1c;
            ent[w * 4 + 2] = r.s0g;
            ent[w * 4 + 3] = r.s1g;
        }
        if (nuniq) {
            nuniq[w * 3 + 0] = r.nc;
            nuniq[w * 3 + 1] = r.ng;
            nuniq[w * 3 + 2] = r.ngf;
        }
        if (mm_key) mm_key[w] = r.best.key;
        if (mm_cnt) mm_cnt[w] = (long long)r.best.cnt;
        if (mm_first) mm_first[w] = r.best.first;
    }
    return 0;
}

// the two historical views of the summary (host outputs)
extern "C" int mpb_hist_stats(mpb_hist* h, int64_t* gap_n, double* ent, int64_t* nuniq, uint64_t* mm_key,
                              int64_t* mm_cnt, uint64_t* mm_first, int64_t* n_iupac_gap) {
    return mpb_hist_summary(h, gap_n, ent, nuniq, mm_key, mm_cnt, mm_first, n_iupac_gap, nullptr, nullptr);
}

// tensors of the windows with sel[i] != 0 only (zeros elsewhere); they also stay on the device for the walk
extern "C" int mpb_hist_tensors(mpb_hist* h, const uint8_t* sel, int64_t* freq_hd, int64_t* nn_hd) {
    if (!h || !sel || !freq_hd || !nn_hd) return fail(MPB_EINVAL, "NULL argument");
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    const int k = h->k;
    const size_t fb = (size_t)h->nw * 4 * k * 8, nb = (size_t)h->nw * (k - 1) * 16 * 8;
    std::vector<int32_t> idx;
    for (int i = 0; i < h->nw; ++i)
        if (sel[i]) idx.push_back(i);
    CK(cudaMemsetAsync(h->freq, 0, fb, ctx->stream));
    CK(cudaMemsetAsync(h->nn, 0, nb, ctx->stream));
    if (!idx.empty()) {
        InBuf si(ctx, idx.data(), idx.size() * 4);
        if (si.rc) return si.rc;
        MPB_LAUNCH_NAMED(ctx, "k_hist_summary", (k_hist_summary<false, true>), dim3(SUM_SB, (unsigned)idx.size()), SUM_THREADS, 0,
                         h->keys, h->cnt, h->first, h->elist, h->n_entries, h->log2cap, k, h->v, si.dev<int32_t>(),
                         (StatsPart*)nullptr, h->freq, h->nn);
    }
    CK(cudaMemcpyAsync(freq_hd, h->freq, fb, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(nn_hd, h->nn, nb, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    h->have_summary = true;
    return 0;
}

__global__ void k_hist_dump(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ cnt,
                            const uint64_t* __restrict__ first, const uint32_t* __restrict__ elist, int log2cap, int wi,
                            long long n, uint64_t* __restrict__ ok, uint32_t* __restrict__ oc, uint64_t* __restrict__ of) {
    const uint64_t base = (uint64_t)wi << log2cap;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const uint64_t slot = base + elist[base + i];
        ok[i] = keys[slot];
        oc[i] = cnt[slot];
        of[i] = first[slot];
    }
}

extern "C" int mpb_hist_dump(mpb_hist* h, int32_t w, int64_t max_n, uint64_t* keys_hd, uint32_t* cnt_hd,
                             uint64_t* first_hd, int64_t* n_out) {
    if (!h || !keys_hd || !cnt_hd || !first_hd || !n_out) return fail(MPB_EINVAL, "NULL argument");
    if (w < 0 || w >= h->nw || max_n < 0) return fail(MPB_EINVAL, "window %d outside the batch", w);
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    unsigned long long n = 0;
    CK(cudaMemcpyAsync(&n, h->n_entries + w, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *n_out = (int64_t)n;
    const long long take = (long long)n < max_n ? (long long)n : max_n;
    if (take <= 0) return 0;
    OutBuf ok(ctx, keys_hd, take * 8), oc(ctx, cnt_hd, take * 4), of(ctx, first_hd, take * 8);
    if (ok.rc || oc.rc || of.rc) return MPB_ENOMEM;
    unsigned grid = (unsigned)((take + 255) / 256);
    if (grid > (unsigned)ctx->sm_count * 8) grid = ctx->sm_count * 8;
    LAUNCH(ctx, k_hist_dump, grid, 256, 0, h->keys, h->cnt, h->first, h->elist, h->log2cap, (int)w, take,
           ok.dev<uint64_t>(), oc.dev<uint32_t>(), of.dev<uint64_t>());
    CK(ok.finish());
    CK(oc.finish());
    CK(of.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// distinct gap-free table entries matched exactly by a degenerate pattern; MATCH_SB blocks per query over the entry list
#define MATCH_SB 4
__global__ void __launch_bounds__(256)
k_hist_match(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ elist,
             const unsigned long long* __restrict__ n_entries, int log2cap, int k, const int32_t* __restrict__ q_win,
             const uint32_t* __restrict__ q_allow, unsigned long long* __restrict__ out) {
    const int q = blockIdx.y;
    const uint64_t base = (uint64_t)q_win[q] << log2cap;
    const long long n_e = (long long)n_entries[q_win[q]];
    const uint32_t kmask = (1u << k) - 1u;
    const uint32_t na = ~q_allow[q * 4 + 0] & kmask, ncm = ~q_allow[q * 4 + 1] & kmask, ngm = ~q_allow[q * 4 + 2] & kmask,
                   nt = ~q_allow[q * 4 + 3] & kmask;
    unsigned n = 0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n_e; i += (long long)gridDim.x * 256) {
        const uint64_t key = keys[base + elist[base + i]];
        if (key >= MPB_KEY_BASE5_D) continue;  // a k-mer with gaps (never an expansion of a primer)
        uint32_t a, c, g, t, gapv;
        mpb_key_planes(key, k, kmask, a, c, g, t, gapv);
        n += ((a & na) | (c & ncm) | (g & ngm) | (t & nt)) == 0u;
    }
    n = __reduce_add_sync(0xffffffffu, n);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(&out[q], (unsigned long long)n);
}

extern "C" int mpb_hist_match(mpb_hist* h, const int32_t* q_win, const uint32_t* q_allow, int32_t nq,
                              int64_t* distinct_hd) {
    if (!h || !q_win || !q_allow || !distinct_hd) return fail(MPB_EINVAL, "NULL argument");
    if (nq < 1) return 0;
    if (!mpb_is_device_ptr(q_win))
        for (int i = 0; i < nq; ++i)
            if (q_win[i] < 0 || q_win[i] >= h->nw) return fail(MPB_EINVAL, "q_win[%d]=%d outside the batch", i, q_win[i]);
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    InBuf qw(ctx, q_win, (size_t)nq * 4), qa(ctx, q_allow, (size_t)nq * 16);
    OutBuf o(ctx, distinct_hd, (size_t)nq * 8);
    if (qw.rc || qa.rc || o.rc) return MPB_ECUDA;
    CK(cudaMemsetAsync(o.d, 0, (size_t)nq * 8, ctx->stream));
    LAUNCH(ctx, k_hist_match, dim3(MATCH_SB, (unsigned)nq), 256, 0, h->keys, h->elist, h->n_entries, h->log2cap, h->k,
           qw.dev<int32_t>(), qa.dev<uint32_t>(), o.dev<unsigned long long>());
    CK(o.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int mpb_hist_exceptions(mpb_hist* h, int64_t max_n, int32_t* win_idx, int32_t* seq_idx, int64_t* n_out) {
    if (!h || !n_out) return fail(MPB_EINVAL, "NULL argument");
    mpb_ctx* ctx = h->msa->ctx;
    CK(cudaSetDevice(ctx->device));
    unsigned long long n = 0;
    CK(cudaMemcpyAsync(&n, h->exc_n, 8, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if ((int64_t)n > h->exc_max) return fail(MPB_EOVERFLOW, "more than %lld IUPAC gap rows in one batch", (long long)h->exc_max);
    *n_out = (int64_t)n;
    int64_t take = (int64_t)n < max_n ? (int64_t)n : max_n;
    if (take > 0 && win_idx && seq_idx) {
        std::vector<int32_t> tmp(2 * take);
        CK(cudaMemcpyAsync(tmp.data(), h->exc, take * 8, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (int64_t i = 0; i < take; ++i) {
            win_idx[i] = tmp[2 * i];
            seq_idx[i] = tmp[2 * i + 1];
        }
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// the candidate scan (mis_primer_check, core:1103-1130)
// ------------------------------------------------------------------------------------------------------
#define SCAN_THREADS 256
#define SCAN_CHUNK 4       // candidates of one window evaluated together against a window held in registers
#define SCAN_MAX_CPB 128   // chunks per block (shared-memory counters: 128*8*3*4 = 12 KB)

// one candidate against one one-hot k-mer: mismatch vector, then the three classes of core:1114-1127
#define SCAN_EVAL(A_, C_, G_, T_, ci)                                                             \
    {                                                                                             \
        const uint32_t mis = w.gapv | ((A_) & nA[ci]) | ((C_) & nC[ci]) | ((G_) & nG[ci]) | ((T_) & nT[ci]); \
        const bool within = __popc(mis) <= v;                                                     \
        const bool okf = within && (mis & fmask) == 0u;                                           \
        const bool okr = within && (mis & rmask) == 0u;                                           \
        acc0[ci] += (mis == 0u);                                                                  \
        accf[ci] += okf; /* includes the perfect matches; they are subtracted after the reduction */ \
        accr[ci] += okr;                                                                          \
        if (BITS) {                                                                               \
            nonf |= (!okf) << ci;                                                                 \
            nonr |= (!okr) << ci;                                                                 \
        }                                                                                         \
    }

#define SCAN_SPECIAL_CAP 3072  // deferred (chunk, row) pairs per block

// One chunk (CNT candidates of one window, masks in registers) against the block's sequence tiles.
// Rows that need more than the funnel shift — the window starts / ends inside a gap run, holds IUPAC cells, or runs
// past a ragged row — are "special" (about 0.5 % of the rows).  Handling them inline left most of the warp idle for
// hundreds of instructions, so when DEFER is set they are only recorded in a
// block-private list and evaluated densely, one per thread, after the block has walked all its chunks.
template <bool BITS, int CNT>
__device__ __forceinline__ void scan_chunk(const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq,
                                           const int32_t* __restrict__ lens, int k, int v, uint32_t kmask,
                                           uint32_t fmask, uint32_t rmask, int first, int p, long long tile0,
                                           int tiles_per_block, const uint32_t* __restrict__ cand_allow,
                                           unsigned int* __restrict__ s_out, const int32_t* __restrict__ bits_slot,
                                           uint32_t* __restrict__ bits, long long words, int* __restrict__ err,
                                           int ch_local, unsigned int* __restrict__ s_special,
                                           unsigned int* __restrict__ s_nspecial) {
    constexpr bool DEFER = !BITS;
    uint32_t nA[CNT], nC[CNT], nG[CNT], nT[CNT];
    unsigned acc0[CNT], accf[CNT], accr[CNT];
#pragma unroll
    for (int ci = 0; ci < CNT; ++ci) {
        const uint4 al = __ldg((const uint4*)(cand_allow) + first + ci);
        nA[ci] = ~al.x & kmask;
        nC[ci] = ~al.y & kmask;
        nG[ci] = ~al.z & kmask;
        nT[ci] = ~al.w & kmask;
        acc0[ci] = accf[ci] = accr[ci] = 0;
    }
    const int lane = threadIdx.x & 31;
    // the two column words of this window: uniform for the whole block
    const uint4* __restrict__ wbase = reinterpret_cast<const uint4*>(pl) + (int64_t)(p >> 5) * nsp;
    const int sh = p & 31;
    for (int t = 0; t < tiles_per_block; ++t) {
        const long long tile = tile0 + t;
        if (tile * SCAN_THREADS >= n_seq) break;  // uniform
        const int64_t s = tile * SCAN_THREADS + threadIdx.x;
        const bool valid = s < n_seq;
        Win w;
        w.a = w.c = w.g = w.t = w.multi = 0;
        w.gapv = kmask;
        bool isgap = false;
        unsigned nonf = 0, nonr = 0;
        if (valid) {
            const uint4 q0 = __ldg(wbase + s), q1 = __ldg(wbase + nsp + s);
            w.a = __funnelshift_r(q0.x, q1.x, sh) & kmask;
            w.c = __funnelshift_r(q0.y, q1.y, sh) & kmask;
            w.g = __funnelshift_r(q0.z, q1.z, sh) & kmask;
            w.t = __funnelshift_r(q0.w, q1.w, sh) & kmask;
            uint32_t gapv = ~(w.a | w.c | w.g | w.t) & kmask;
            const int len = lens[s];
            const bool ragged = p + k > len;
            const bool edge = (((gapv & 1u) | ((gapv >> (k - 1)) & 1u)) != 0u) && gapv != kmask;
            w.multi = mpb_multi(w.a, w.c, w.g, w.t);
            bool special = ragged || edge || w.multi != 0u;
            if (DEFER && special) {
                const unsigned slot = atomicAdd(s_nspecial, 1u);
                if (slot < SCAN_SPECIAL_CAP) {
                    s_special[slot] = ((unsigned)ch_local << 16) | (unsigned)(t * SCAN_THREADS + threadIdx.x);
                } else {
                    special = true;  // list full: fall through to the inline path below
                    atomicSub(s_nspecial, 1u);
                }
                if (slot < SCAN_SPECIAL_CAP) goto next_tile;
            }
            if (special) {
                if (ragged) {
                    Win tmp;
                    if (!mpb_window_slow(pl, nsp, s, len, p, k, tmp)) atomicOr(err, MPB_ERR_SHORT_ROW);
                    w.a = tmp.a;
                    w.c = tmp.c;
                    w.g = tmp.g;
                    w.t = tmp.t;
                } else if (edge) {
                    mpb_patch_edges(pl, nsp, s, len, p, k, kmask, w);
                }
                gapv = ~(w.a | w.c | w.g | w.t) & kmask;
                w.multi = mpb_multi(w.a, w.c, w.g, w.t);
            }
            w.gapv = gapv;
            isgap = __popc(gapv) > v;
            if (!isgap) {
                if (w.multi == 0) {
#pragma unroll
                    for (int ci = 0; ci < CNT; ++ci) SCAN_EVAL(w.a, w.c, w.g, w.t, ci)
                } else {
                    const uint32_t nexp = mpb_expansions(w);
                    if (nexp > MPB_MAX_EXP) {
                        atomicOr(err, MPB_ERR_EXPAND);
                    } else {
                        for (uint32_t e = 0; e < nexp; ++e) {
                            uint32_t a, c, g, tt;
                            mpb_expand(w, e, a, c, g, tt);
#pragma unroll
                            for (int ci = 0; ci < CNT; ++ci) SCAN_EVAL(a, c, g, tt, ci)
                        }
                    }
                }
            }
        }
    next_tile:
        if (BITS) {
            const long long word = tile * (SCAN_THREADS / 32) + (threadIdx.x >> 5);
            const unsigned bg = __ballot_sync(0xffffffffu, isgap);
#pragma unroll
            for (int ci = 0; ci < CNT; ++ci) {
                const int slot = bits_slot[first + ci];
                if (slot < 0) continue;  // uniform
                const unsigned bf = __ballot_sync(0xffffffffu, (nonf >> ci) & 1u);
                const unsigned br = __ballot_sync(0xffffffffu, (nonr >> ci) & 1u);
                if (lane == 0 && word < words) {
                    uint32_t* o = bits + (long long)slot * 3 * words;
                    o[word] = bf;
                    o[words + word] = br;
                    o[2 * words + word] = bg;
                }
            }
        }
    }
#pragma unroll
    for (int ci = 0; ci < CNT; ++ci) {
        const unsigned r0 = __reduce_add_sync(0xffffffffu, acc0[ci]);
        const unsigned rf = __reduce_add_sync(0xffffffffu, accf[ci]) - r0;   // 1..v mismatches only
        const unsigned rr = __reduce_add_sync(0xffffffffu, accr[ci]) - r0;
        if (lane < 3) {
            const unsigned val = lane == 0 ? r0 : (lane == 1 ? rf : rr);
            if (val) atomicAdd(&s_out[ci * 3 + lane], val);
        }
    }
}

// the deferred rows of a block: one (chunk, row) pair per thread, full window logic, shared-memory counters
__device__ __forceinline__ void scan_special(const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq,
                                             const int32_t* __restrict__ lens, int k, int v, uint32_t kmask,
                                             uint32_t fmask, uint32_t rmask, const int4* __restrict__ chunks, int ch0,
                                             long long tile0, const uint32_t* __restrict__ cand_allow,
                                             unsigned int* __restrict__ s_cnt, const unsigned int* __restrict__ s_special,
                                             unsigned int n_special, int* __restrict__ err) {
    for (unsigned i = threadIdx.x; i < n_special; i += SCAN_THREADS) {
        const unsigned e = s_special[i];
        const int ch_local = (int)(e >> 16);
        const int4 cd = chunks[ch0 + ch_local];
        const int64_t s = tile0 * SCAN_THREADS + (e & 0xFFFFu);
        Win w;
        if (!mpb_load_window(pl, nsp, s, lens[s], cd.z, k, kmask, w)) atomicOr(err, MPB_ERR_SHORT_ROW);
        if (__popc(w.gapv) > v) continue;  // gap row: no contribution
        uint32_t nexp = 1;
        if (w.multi) {
            nexp = mpb_expansions(w);
            if (nexp > MPB_MAX_EXP) {
                atomicOr(err, MPB_ERR_EXPAND);
                continue;
            }
        }
        for (int ci = 0; ci < cd.y; ++ci) {
            const uint4 al = __ldg((const uint4*)(cand_allow) + cd.x + ci);
            const uint32_t nA = ~al.x & kmask, nC = ~al.y & kmask, nG = ~al.z & kmask, nT = ~al.w & kmask;
            unsigned n0 = 0, nf = 0, nr = 0;
            for (uint32_t x = 0; x < nexp; ++x) {
                uint32_t a = w.a, c = w.c, g = w.g, tt = w.t;
                if (w.multi) mpb_expand(w, x, a, c, g, tt);
                const uint32_t mis = w.gapv | (a & nA) | (c & nC) | (g & nG) | (tt & nT);
                const bool within = __popc(mis) <= v;
                const bool z = mis == 0u;
                n0 += z;
                nf += within && (mis & fmask) == 0u && !z;
                nr += within && (mis & rmask) == 0u && !z;
            }
            unsigned int* o = &s_cnt[(ch_local * SCAN_CHUNK + ci) * 3];
            if (n0) atomicAdd(&o[0], n0);
            if (nf) atomicAdd(&o[1], nf);
            if (nr) atomicAdd(&o[2], nr);
        }
    }
}

// Block (x, y): sequences [x*T*256, (x+1)*T*256) against the chunks [y*cpb, (y+1)*cpb).  A chunk = up to
// SCAN_CHUNK candidates of ONE window: their masks sit in registers while the block walks its T sequence tiles
// (T small enough that the tiles' words stay in L1 for the next chunk of the same column word), each thread keeping
// per-candidate counters in registers; one warp reduction per chunk, block-private counters in shared memory, one
// coalesced store of the block's partial counts at the end (no global atomics).
template <bool BITS>
__global__ void __launch_bounds__(SCAN_THREADS, 4)
k_scan(const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq, const int32_t* __restrict__ lens, int k, int v,
       uint32_t fmask, uint32_t rmask, const int4* __restrict__ chunks, int n_chunks, int cpb, int tiles_per_block,
       const uint32_t* __restrict__ cand_allow, uint32_t* __restrict__ partial, long long nc,
       const int32_t* __restrict__ bits_slot, uint32_t* __restrict__ bits, long long words, int* __restrict__ err) {
    __shared__ unsigned int s_cnt[SCAN_MAX_CPB * SCAN_CHUNK * 3];
    __shared__ unsigned int s_special[BITS ? 1 : SCAN_SPECIAL_CAP];
    __shared__ unsigned int s_nspecial;
    const int ch0 = blockIdx.y * cpb;
    const int ch1 = min(n_chunks, ch0 + cpb);
    for (int i = threadIdx.x; i < (ch1 - ch0) * SCAN_CHUNK * 3; i += SCAN_THREADS) s_cnt[i] = 0;
    if (threadIdx.x == 0) s_nspecial = 0;
    __syncthreads();
    const uint32_t kmask = (1u << k) - 1u;
    const long long tile0 = (long long)blockIdx.x * tiles_per_block;
    for (int ch = ch0; ch < ch1; ++ch) {
        const int4 cd = chunks[ch];  // first candidate, count, window column
        unsigned int* so = &s_cnt[(ch - ch0) * SCAN_CHUNK * 3];
        switch (cd.y) {
            case 1:
                scan_chunk<BITS, 1>(pl, nsp, n_seq, lens, k, v, kmask, fmask, rmask, cd.x, cd.z, tile0, tiles_per_block,
                                    cand_allow, so, bits_slot, bits, words, err, ch - ch0, s_special, &s_nspecial);
                break;
            case 2:
                scan_chunk<BITS, 2>(pl, nsp, n_seq, lens, k, v, kmask, fmask, rmask, cd.x, cd.z, tile0, tiles_per_block,
                                    cand_allow, so, bits_slot, bits, words, err, ch - ch0, s_special, &s_nspecial);
                break;
            case 3:
                scan_chunk<BITS, 3>(pl, nsp, n_seq, lens, k, v, kmask, fmask, rmask, cd.x, cd.z, tile0, tiles_per_block,
                                    cand_allow, so, bits_slot, bits, words, err, ch - ch0, s_special, &s_nspecial);
                break;
            default:
                scan_chunk<BITS, 4>(pl, nsp, n_seq, lens, k, v, kmask, fmask, rmask, cd.x, cd.z, tile0, tiles_per_block,
                                    cand_allow, so, bits_slot, bits, words, err, ch - ch0, s_special, &s_nspecial);
                break;
        }
    }
    __syncthreads();
    if (!BITS) {
        scan_special(pl, nsp, n_seq, lens, k, v, kmask, fmask, rmask, chunks, ch0, tile0, cand_allow, s_cnt, s_special,
                     s_nspecial, err);
        __syncthreads();
    }
    // partial[x][candidate][3]
    uint32_t* out = partial + (long long)blockIdx.x * nc * 3;
    for (int ch = ch0; ch < ch1; ++ch) {
        const int4 cd = chunks[ch];
        for (int i = threadIdx.x; i < cd.y * 3; i += SCAN_THREADS)
            out[(long long)cd.x * 3 + i] = s_cnt[(ch - ch0) * SCAN_CHUNK * 3 + i];
    }
}

__global__ void k_scan_reduce(const uint32_t* __restrict__ partial, int gx, long long n3,
                              unsigned long long* __restrict__ counts) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n3) return;
    unsigned long long acc = 0;
    for (int x = 0; x < gx; ++x) acc += partial[(long long)x * n3 + i];
    counts[i] = acc;
}

extern "C" int mpb_scan(mpb_msa* m, int k, int v, uint32_t fmask, uint32_t rmask, const int32_t* cand_pos_hd,
                        const uint32_t* cand_allow_hd, int64_t nc, int64_t* counts_hd, const int32_t* bits_slot,
                        uint32_t* bits_hd) {
    if (!m || !cand_pos_hd || !cand_allow_hd || !counts_hd) return fail(MPB_EINVAL, "NULL argument");
    if (k < 3 || k > MPB_MAX_K) return fail(MPB_EINVAL, "primer length %d outside 3..%d", k, MPB_MAX_K);
    if (nc < 1) return 0;
    if (nc >= (1ll << 31) / 4) return fail(MPB_EINVAL, "too many candidates in one call");
    if (bits_slot && !bits_hd) return fail(MPB_EINVAL, "bits_slot without bits");
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    const long long words = (m->n_seq + 31) / 32;
    // candidate windows are needed on the host to cut the chunks
    std::vector<int32_t> pos_copy;
    const int32_t* pos = cand_pos_hd;
    if (mpb_is_device_ptr(cand_pos_hd)) {
        pos_copy.resize(nc);
        CK(cudaMemcpyAsync(pos_copy.data(), cand_pos_hd, nc * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        pos = pos_copy.data();
    }
    std::vector<int4> chunks;
    for (int64_t i = 0; i < nc;) {
        if (pos[i] < 0 || pos[i] >= m->n_col)
            return fail(MPB_EINVAL, "cand_pos[%lld]=%d outside the alignment", (long long)i, pos[i]);
        int64_t j = i + 1;
        while (j < nc && j - i < SCAN_CHUNK && pos[j] == pos[i]) ++j;
        chunks.push_back(make_int4((int)i, (int)(j - i), pos[i], 0));
        i = j;
    }
    int nslots = 0;
    if (bits_slot)
        for (int64_t i = 0; i < nc; ++i)
            if (bits_slot[i] >= nslots) nslots = bits_slot[i] + 1;
    const int n_chunks = (int)chunks.size();
    const long long n_tiles = (m->n_seq + SCAN_THREADS - 1) / SCAN_THREADS;
    const long long target = (long long)ctx->sm_count * 8;  // blocks in flight we want at least
    int tpb = (int)(n_tiles * n_chunks / (target * 16));     // tiles per block: long walks amortise the reductions
    if (tpb < 1) tpb = 1;
    if (tpb > 4) tpb = 4;  // 4 CTAs/SM x 4 tiles x 8 KB of window words stay L1-resident across chunks
    const int gx = (int)((n_tiles + tpb - 1) / tpb);
    int cpb = (int)(((long long)n_chunks * gx + target - 1) / target);
    if (cpb < 1) cpb = 1;
    if (cpb > SCAN_MAX_CPB) cpb = SCAN_MAX_CPB;
    const int gy = (n_chunks + cpb - 1) / cpb;
    InBuf ca(ctx, cand_allow_hd, (size_t)nc * 16), bs(ctx, bits_slot, (size_t)nc * 4),
        chk(ctx, chunks.data(), chunks.size() * sizeof(int4));
    OutBuf oc(ctx, counts_hd, (size_t)nc * 3 * 8), ob(ctx, bits_hd, (size_t)nslots * 3 * words * 4);
    if (ca.rc || bs.rc || chk.rc || oc.rc || ob.rc) return MPB_ECUDA;
    uint32_t* partial = nullptr;
    CK(cudaMallocAsync(&partial, (size_t)gx * nc * 3 * 4, ctx->stream));
    dim3 grid((unsigned)gx, (unsigned)gy);
    ctx->pending_units = (double)nc * (double)m->n_seq;  // candidate x sequence evaluations of this launch
    if (bits_slot) {
        LAUNCH(ctx, k_scan<true>, grid, SCAN_THREADS, 0, m->planes, m->nsp, m->n_seq, m->lens, k, v, fmask, rmask,
               chk.dev<int4>(), n_chunks, cpb, tpb, ca.dev<uint32_t>(), partial, (long long)nc, bs.dev<int32_t>(),
               ob.dev<uint32_t>(), words, m->err);
    } else {
        LAUNCH(ctx, k_scan<false>, grid, SCAN_THREADS, 0, m->planes, m->nsp, m->n_seq, m->lens, k, v, fmask, rmask,
               chk.dev<int4>(), n_chunks, cpb, tpb, ca.dev<uint32_t>(), partial, (long long)nc, (const int32_t*)nullptr,
               (uint32_t*)nullptr, words, m->err);
    }
    LAUNCH(ctx, k_scan_reduce, (unsigned)((nc * 3 + 255) / 256), 256, 0, partial, gx, (long long)nc * 3,
           oc.dev<unsigned long long>());
    CK(cudaFreeAsync(partial, ctx->stream));
    CK(oc.finish());
    CK(ob.finish());
    return mpb_check_flags(ctx, m->err);  // also keeps the host chunk list alive until the kernels are done
}

// per (window, sequence) table key, for the JSON side files
__global__ void k_seqkeys(const uint32_t* __restrict__ pl, int64_t nsp, int64_t n_seq, const int32_t* __restrict__ lens,
                          int k, const int32_t* __restrict__ win_pos, int nw, uint64_t* __restrict__ out) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seq) return;
    const uint32_t kmask = (1u << k) - 1u;
    const int len = lens[s];
    for (int wi = blockIdx.y; wi < nw; wi += gridDim.y) {
        Win w;
        mpb_load_window(pl, nsp, s, len, win_pos[wi], k, kmask, w);
        out[(int64_t)wi * n_seq + s] = w.multi ? MPB_KEY_IUPAC_D : mpb_key(w.c, w.g, w.t, w.gapv, k);
    }
}

extern "C" int mpb_seqkeys(mpb_msa* m, int k, const int32_t* win_pos, int32_t nw, uint64_t* out_hd) {
    if (!m || !win_pos || !out_hd) return fail(MPB_EINVAL, "NULL argument");
    if (k < 3 || k > MPB_MAX_K || nw < 1) return fail(MPB_EINVAL, "bad k=%d or nw=%d", k, nw);
    mpb_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    InBuf wp(ctx, win_pos, (size_t)nw * 4);
    OutBuf o(ctx, out_hd, (size_t)nw * m->n_seq * 8);
    if (wp.rc || o.rc) return MPB_ECUDA;
    unsigned gx = (unsigned)((m->n_seq + 255) / 256), gy = (unsigned)nw;
    if (gy > 1024) gy = 1024;
    LAUNCH(ctx, k_seqkeys, dim3(gx, gy), 256, 0, m->planes, m->nsp, m->n_seq, m->lens, k, wp.dev<int32_t>(), nw,
           o.dev<uint64_t>());
    CK(o.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// nearest-neighbour Tm (core:249-261, 328-335).  The 4x4 dH / dS tables and the initiation terms are staged
// into shared memory with one TMA bulk copy (cp.async.bulk) per CTA, completion on an mbarrier.
// ------------------------------------------------------------------------------------------------------
// [0..15] dH[next][cur], [16..31] dS[next][cur], [32..35] dH init (A,C,G,T), [36..39] dS init
__device__ __align__(16) double g_nn_tables[40] = {
    -7.9, -8.5, -8.2, -7.2, -8.4, -8.0, -9.8, -8.2, -7.8, -10.6, -8.0, -8.5, -7.2, -7.8, -8.4, -7.9,
    -22.2, -22.7, -22.2, -21.3, -22.4, -19.9, -24.4, -22.2, -21.0, -27.2, -19.9, -22.7, -20.4, -21.0, -22.4, -22.2,
    2.3, 0.1, 0.1, 2.3, 4.1, -2.8, -2.8, 4.1};

__global__ void __launch_bounds__(128)
k_tm(const uint8_t* __restrict__ seqs, int k, long long n, double c_nonsym, double c_sym, double corr,
     double* __restrict__ tm, double* __restrict__ dh_out, double* __restrict__ ds_out) {
    __shared__ __align__(16) double tab[40];
    __shared__ __align__(8) unsigned long long bar;
    const unsigned bar_addr = (unsigned)__cvta_generic_to_shared(&bar);
    const unsigned tab_addr = (unsigned)__cvta_generic_to_shared(tab);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_addr));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_addr), "r"(320u) : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(tab_addr),
            "l"(g_nn_tables), "r"(320u), "r"(bar_addr)
            : "memory");
    }
    {
        unsigned done = 0;
        while (!done) {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                "selp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(bar_addr), "r"(0u)
                : "memory");
        }
    }
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* q = seqs + i * k;
    // left-to-right sums starting from 0, exactly the reference's operation order; no FMA contraction
    double dh = 0.0, ds = 0.0;
    for (int j = 0; j + 1 < k; ++j) {
        const int nx = q[j + 1], cu = q[j];
        dh = __dadd_rn(dh, tab[nx * 4 + cu]);
        ds = __dadd_rn(ds, tab[16 + nx * 4 + cu]);
    }
    dh = __dadd_rn(dh, __dadd_rn(tab[32 + q[0]], tab[32 + q[k - 1]]));
    ds = __dadd_rn(ds, __dadd_rn(tab[36 + q[0]], tab[36 + q[k - 1]]));
    bool sym = (k % 2) == 0;
    for (int j = 0; sym && j < k / 2; ++j) sym = (q[j] + q[k / 2 + j]) == 3;  // first half == complement(second half)
    if (sym) ds = __dadd_rn(ds, -1.4);
    dh = __dmul_rn(dh, 1000.0);
    const double denom = __dadd_rn(ds, sym ? c_sym : c_nonsym);
    const double t = __dadd_rn(__ddiv_rn(1.0, __dadd_rn(__ddiv_rn(1.0, __ddiv_rn(dh, denom)), corr)), -273.15);
    tm[i] = t;
    if (dh_out) dh_out[i] = dh;
    if (ds_out) ds_out[i] = ds;
}

extern "C" int mpb_tm(mpb_ctx* ctx, const uint8_t* seqs_hd, int k, int64_t n, const double* consts3, double* tm_hd,
                      double* dh_hd, double* ds_hd) {
    if (!ctx || !seqs_hd || !consts3 || !tm_hd) return fail(MPB_EINVAL, "NULL argument");
    if (k < 2 || n < 0) return fail(MPB_EINVAL, "bad k=%d n=%lld", k, (long long)n);
    if (n == 0) return 0;
    CK(cudaSetDevice(ctx->device));
    InBuf in(ctx, seqs_hd, (size_t)n * k);
    OutBuf ot(ctx, tm_hd, n * 8), oh(ctx, dh_hd, n * 8), os(ctx, ds_hd, n * 8);
    if (in.rc || ot.rc || oh.rc || os.rc) return MPB_ECUDA;
    LAUNCH(ctx, k_tm, (unsigned)((n + 127) / 128), 128, 0, in.dev<uint8_t>(), k, (long long)n, consts3[0], consts3[1],
           consts3[2], ot.dev<double>(), oh.dev<double>(), os.dev<double>());
    CK(ot.finish());
    CK(oh.finish());
    CK(os.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// Tm of a degenerate primer = mean over its expansions of the per-expansion Tm rounded to 2 decimals (core:849-852).
// One block per primer; a thread decodes its expansions straight from the base sets (no host enumeration, no H2D of
// expansion strings), evaluates Tm in the reference's operation order (as k_tm) and rounds it to integer hundredths;
// the block adds the integers — exact and order-independent.  An expansion whose Tm sits within 1e-6 of a rounding tie
// is counted in `ties`: the caller then replays that primer on the host with Python's round().
__global__ void __launch_bounds__(128)
k_tm_sets(const uint8_t* __restrict__ sets, int k, int n, double c_nonsym, double c_sym, double corr,
          long long* __restrict__ sums, int* __restrict__ ties) {
    __shared__ __align__(16) double tab[40];
    __shared__ long long s_sum;
    __shared__ int s_tie;
    for (int i = threadIdx.x; i < 40; i += blockDim.x) tab[i] = g_nn_tables[i];
    if (threadIdx.x == 0) {
        s_sum = 0;
        s_tie = 0;
    }
    __syncthreads();
    const int pi = blockIdx.x;
    if (pi >= n) return;
    const uint8_t* S = sets + (long long)pi * 32;
    long long deg = 1;
    for (int i = 0; i < k; ++i) deg *= c_fold[S[i] & 15];
    long long acc = 0;
    int tie = 0;
    for (long long e0 = threadIdx.x; e0 < deg; e0 += blockDim.x) {
        uint8_t q[MPB_MAX_K + 5];
        long long e = e0;
        for (int i = k - 1; i >= 0; --i) {
            const int code = S[i] & 15;
            const int f = c_fold[code];
            q[i] = (uint8_t)((c_order[code] >> (2 * (int)(e % f))) & 3);
            e /= f;
        }
        double dh = 0.0, ds = 0.0;
        for (int j = 0; j + 1 < k; ++j) {
            const int nx = q[j + 1], cu = q[j];
            dh = __dadd_rn(dh, tab[nx * 4 + cu]);
            ds = __dadd_rn(ds, tab[16 + nx * 4 + cu]);
        }
        dh = __dadd_rn(dh, __dadd_rn(tab[32 + q[0]], tab[32 + q[k - 1]]));
        ds = __dadd_rn(ds, __dadd_rn(tab[36 + q[0]], tab[36 + q[k - 1]]));
        bool sym = (k % 2) == 0;
        for (int j = 0; sym && j < k / 2; ++j) sym = (q[j] + q[k / 2 + j]) == 3;
        if (sym) ds = __dadd_rn(ds, -1.4);
        dh = __dmul_rn(dh, 1000.0);
        const double denom = __dadd_rn(ds, sym ? c_sym : c_nonsym);
        const double t = __dadd_rn(__ddiv_rn(1.0, __dadd_rn(__ddiv_rn(1.0, __ddiv_rn(dh, denom)), corr)), -273.15);
        const double y = __dmul_rn(t, 100.0);
        const double fl = floor(y);
        const double fr = y - fl;
        if (fr < 0.5 - 1e-6) acc += (long long)fl;
        else if (fr > 0.5 + 1e-6) acc += (long long)fl + 1;
        else ++tie;
    }
    atomicAdd((unsigned long long*)&s_sum, (unsigned long long)acc);
    if (tie) atomicAdd(&s_tie, tie);
    __syncthreads();
    if (threadIdx.x == 0) {
        sums[pi] = s_sum;
        ties[pi] = s_tie;
    }
}

// sums[n]: sum over the expansions of round(Tm, 2) in hundredths; ties[n]: expansions left out because they sit on a
// rounding tie (host outputs)
extern "C" int mpb_tm_sets(mpb_ctx* ctx, const uint8_t* sets_hd, int k, int32_t n, const double* consts3, int64_t* sums,
                           int32_t* ties) {
    if (!ctx || !sets_hd || !consts3 || !sums || !ties) return fail(MPB_EINVAL, "NULL argument");
    if (k < 2 || k > MPB_MAX_K || n < 0) return fail(MPB_EINVAL, "bad k=%d n=%d", k, n);
    if (n == 0) return 0;
    CK(cudaSetDevice(ctx->device));
    InBuf in(ctx, sets_hd, (size_t)n * 32);
    OutBuf os(ctx, sums, (size_t)n * 8), ot(ctx, ties, (size_t)n * 4);
    if (in.rc || os.rc || ot.rc) return MPB_ECUDA;
    LAUNCH(ctx, k_tm_sets, (unsigned)n, 128, 0, in.dev<uint8_t>(), k, (int)n, consts3[0], consts3[1], consts3[2],
           os.dev<long long>(), ot.dev<int>());
    CK(os.finish());
    CK(ot.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// ------------------------------------------------------------------------------------------------------
// pair coverage (get_multiPrime.py:560-569): the sequences NOT covered by a primer pair are the union of the forward
// primer's and the reverse primer's uncovered sets; with per-sequence bit vectors that is popcount(F | R).
// ------------------------------------------------------------------------------------------------------
__global__ void k_pair_cover(const uint32_t* __restrict__ uf, const uint32_t* __restrict__ ur,
                             const int32_t* __restrict__ pf, const int32_t* __restrict__ pr, long long n_pairs,
                             int words, int32_t* __restrict__ out) {
    const long long q = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // warp per pair
    const int lane = threadIdx.x & 31;
    if (q >= n_pairs) return;
    const uint32_t* a = uf + (long long)pf[q] * words;
    const uint32_t* b = ur + (long long)pr[q] * words;
    int n = 0;
    for (int w = lane; w < words; w += 32) n += __popc(a[w] | b[w]);
    n = __reduce_add_sync(0xffffffffu, n);
    if (lane == 0) out[q] = n;
}

extern "C" int mpb_pair_cover(mpb_ctx* ctx, const uint32_t* uf_hd, const uint32_t* ur_hd, int32_t n_rows, int32_t words,
                              const int32_t* pf_hd, const int32_t* pr_hd, int64_t n_pairs, int32_t* uncovered_hd) {
    if (!ctx || !uf_hd || !ur_hd || !pf_hd || !pr_hd || !uncovered_hd) return fail(MPB_EINVAL, "NULL argument");
    if (n_pairs < 1) return 0;
    CK(cudaSetDevice(ctx->device));
    InBuf uf(ctx, uf_hd, (size_t)n_rows * words * 4), ur(ctx, ur_hd, (size_t)n_rows * words * 4),
        pf(ctx, pf_hd, (size_t)n_pairs * 4), pr(ctx, pr_hd, (size_t)n_pairs * 4);
    OutBuf o(ctx, uncovered_hd, (size_t)n_pairs * 4);
    if (uf.rc || ur.rc || pf.rc || pr.rc || o.rc) return MPB_ECUDA;
    LAUNCH(ctx, k_pair_cover, (unsigned)((n_pairs * 32 + 255) / 256), 256, 0, uf.dev<uint32_t>(), ur.dev<uint32_t>(),
           pf.dev<int32_t>(), pr.dev<int32_t>(), (long long)n_pairs, (int)words, o.dev<int32_t>());
    CK(o.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// The same straight from the scan's bit vectors (mpb_cscan / mpb_scan layout bits[row][3][words]: F non-cover, R
// non-cover, gap rows): the forward use of candidate pf leaves F | gap uncovered, the reverse use of pr leaves R | gap
// (get_multiPrime.py:556-569 on the ids of the two JSON side files).  No JSON round trip: SURVEY.md 8f-1.
__global__ void k_pair_cover3(const uint32_t* __restrict__ bits, const int32_t* __restrict__ pf,
                              const int32_t* __restrict__ pr, long long n_pairs, long long words,
                              int32_t* __restrict__ out) {
    const long long q = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // warp per pair
    const int lane = threadIdx.x & 31;
    if (q >= n_pairs) return;
    const uint32_t* a = bits + (long long)pf[q] * 3 * words;
    const uint32_t* b = bits + (long long)pr[q] * 3 * words;
    int n = 0;
    for (long long w = lane; w < words; w += 32) n += __popc(a[w] | a[2 * words + w] | b[words + w] | b[2 * words + w]);
    n = __reduce_add_sync(0xffffffffu, n);
    if (lane == 0) out[q] = n;
}

extern "C" int mpb_pair_cover3(mpb_ctx* ctx, const uint32_t* bits_hd, int32_t n_rows, int64_t words, const int32_t* pf_hd,
                               const int32_t* pr_hd, int64_t n_pairs, int32_t* uncovered_hd) {
    if (!ctx || !bits_hd || !pf_hd || !pr_hd || !uncovered_hd) return fail(MPB_EINVAL, "NULL argument");
    if (n_pairs < 1) return 0;
    CK(cudaSetDevice(ctx->device));
    InBuf bt(ctx, bits_hd, (size_t)n_rows * 3 * words * 4), pf(ctx, pf_hd, (size_t)n_pairs * 4), pr(ctx, pr_hd, (size_t)n_pairs * 4);
    OutBuf o(ctx, uncovered_hd, (size_t)n_pairs * 4);
    if (bt.rc || pf.rc || pr.rc || o.rc) return MPB_ECUDA;
    ctx->pending_units = (double)n_pairs;
    LAUNCH(ctx, k_pair_cover3, (unsigned)((n_pairs * 32 + 255) / 256), 256, 0, bt.dev<uint32_t>(), pf.dev<int32_t>(),
           pr.dev<int32_t>(), (long long)n_pairs, (long long)words, o.dev<int32_t>());
    CK(o.finish());
    CK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

