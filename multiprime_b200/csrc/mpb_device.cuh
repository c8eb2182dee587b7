// mpb_device.cuh — device-side building blocks shared by every kernel of libmpb200:
//   * the bit-plane view of one k-column window of one sequence (with the reference's terminal-gap patching,
//     core:666-687, restated for bit-planes),
//   * IUPAC expansion in the reference's product order (core:105-107, 368-380),
//   * 64-bit haplotype keys and the open-addressing table insert.
// sm_90a only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define MPB_KEY_EMPTY_D 0xFFFFFFFFFFFFFFFFull
#define MPB_KEY_IUPAC_D 0xFFFFFFFFFFFFFFFEull
#define MPB_KEY_BASE5_D (1ull << 54)
#define MPB_ERR_TABLE_FULL 1
#define MPB_ERR_EXPAND 2
#define MPB_ERR_SHORT_ROW 4
#define MPB_MAX_EXP 65536u

// fold (number of alternatives) and expansion order of each 4-bit base set (A=1,C=2,G=4,T=8).
// order byte: alternative j is base ((byte >> 2j) & 3), bases A,C,G,T = 0..3.  core:105-107:
//   R(5)=A,G  Y(10)=C,T  M(3)=A,C  K(12)=G,T  S(6)=G,C  W(9)=A,T  H(11)=A,T,C  B(14)=G,T,C  V(7)=G,A,C
//   D(13)=G,A,T  N(15)=A,T,G,C
static __constant__ uint8_t c_fold[16] = {1, 1, 1, 2, 1, 2, 2, 3, 1, 2, 2, 3, 2, 3, 3, 4};
#define ORD2(a, b) ((a) | ((b) << 2))
#define ORD3(a, b, c) ((a) | ((b) << 2) | ((c) << 4))
#define ORD4(a, b, c, d) ((a) | ((b) << 2) | ((c) << 4) | ((d) << 6))
static __constant__ uint8_t c_order[16] = {
    0,              // 0  gap
    0,              // 1  A
    1,              // 2  C
    ORD2(0, 1),     // 3  M = A,C
    2,              // 4  G
    ORD2(0, 2),     // 5  R = A,G
    ORD2(2, 1),     // 6  S = G,C
    ORD3(2, 0, 1),  // 7  V = G,A,C
    3,              // 8  T
    ORD2(0, 3),     // 9  W = A,T
    ORD2(1, 3),     // 10 Y = C,T
    ORD3(0, 3, 1),  // 11 H = A,T,C
    ORD2(2, 3),     // 12 K = G,T
    ORD3(2, 0, 3),  // 13 D = G,A,T
    ORD3(2, 3, 1),  // 14 B = G,T,C
    ORD4(0, 3, 2, 1)  // 15 N = A,T,G,C
};
static __constant__ uint64_t c_pow5[28] = {1ull,
                                    5ull,
                                    25ull,
                                    125ull,
                                    625ull,
                                    3125ull,
                                    15625ull,
                                    78125ull,
                                    390625ull,
                                    1953125ull,
                                    9765625ull,
                                    48828125ull,
                                    244140625ull,
                                    1220703125ull,
                                    6103515625ull,
                                    30517578125ull,
                                    152587890625ull,
                                    762939453125ull,
                                    3814697265625ull,
                                    19073486328125ull,
                                    95367431640625ull,
                                    476837158203125ull,
                                    2384185791015625ull,
                                    11920928955078125ull,
                                    59604644775390625ull,
                                    298023223876953125ull,
                                    1490116119384765625ull,
                                    7450580596923828125ull};

// One window of one sequence: bit i of plane X is set when the cell at window position i holds base X.
struct Win {
    uint32_t a, c, g, t;  // base planes (an IUPAC cell sets several)
    uint32_t gapv;        // cells without any base
    uint32_t multi;       // cells with more than one base (IUPAC)
};

__device__ __forceinline__ uint32_t mpb_multi(uint32_t a, uint32_t c, uint32_t g, uint32_t t) {
    return (a & c) | (g & t) | ((a ^ c) & (g ^ t));
}

// planes[col_word][seq] = uint4{A, C, G, T}: the four plane words of one sequence and one 32-column word sit in one
// 16-byte vector, so a window costs two coalesced 128-bit loads; one zero word is appended after the last column word
// so that word j+1 exists.
__device__ __forceinline__ uint4 mpb_word(const uint32_t* __restrict__ pl, int64_t nsp, int64_t s, int cw) {
    return __ldg(reinterpret_cast<const uint4*>(pl) + (int64_t)cw * nsp + s);
}

__device__ __forceinline__ int mpb_cell(const uint32_t* __restrict__ pl, int64_t nsp, int64_t s, int col) {
    const uint4 w = mpb_word(pl, nsp, s, col >> 5);
    int b = col & 31;
    return ((w.x >> b) & 1u) | (((w.y >> b) & 1u) << 1) | (((w.z >> b) & 1u) << 2) | (((w.w >> b) & 1u) << 3);
}

// The rare path of core:666-687: the window starts/ends inside a gap run, or runs past the end of a ragged row.
// Restated on an array of k 4-bit cells; returns false when the row cannot supply k cells (unsupported input).
static __device__ __noinline__ bool mpb_window_slow(const uint32_t* __restrict__ pl, int64_t nsp, int64_t s, int len, int p,
                                            int k, Win& out) {
    uint8_t w[32];
    uint8_t buf[32];
    int m = len - p;
    m = m < 0 ? 0 : (m > k ? k : m);
    bool allgap = true;
    for (int i = 0; i < m; ++i) {
        w[i] = (uint8_t)mpb_cell(pl, nsp, s, p + i);
        allgap = allgap && (w[i] == 0);
    }
    const int left_end = p < len ? p : len;  // S[0:p]
    if (!(m == k && allgap)) {
        if (m > 0 && w[0] == 0) {  // leading gap run <- last g bases left of the window
            int g = 0;
            while (g < m && w[g] == 0) ++g;
            int got = 0;
            for (int col = left_end - 1; col >= 0 && got < g; --col) {
                int x = mpb_cell(pl, nsp, s, col);
                if (x) buf[got++] = (uint8_t)x;
            }
            if (got == g)
                for (int i = 0; i < g; ++i) w[i] = buf[g - 1 - i];
        }
        if (m > 0 && w[m - 1] == 0) {  // trailing gap run <- first g bases right of the window
            int g = 0;
            while (g < m && w[m - 1 - g] == 0) ++g;
            int got = 0;
            for (int col = p + k; col < len && got < g; ++col) {
                int x = mpb_cell(pl, nsp, s, col);
                if (x) buf[got++] = (uint8_t)x;
            }
            if (got == g)
                for (int i = 0; i < g; ++i) w[m - g + i] = buf[i];
        }
    }
    bool ok = true;
    if (m < k) {  // ragged row shorter than the window: left-extend (core:683-687)
        int g = k - m;
        int got = 0;
        for (int col = left_end - 1; col >= 0 && got < g; --col) {
            int x = mpb_cell(pl, nsp, s, col);
            if (x) buf[got++] = (uint8_t)x;
        }
        if (got == g) {
            for (int i = m - 1; i >= 0; --i) w[i + g] = w[i];
            for (int i = 0; i < g; ++i) w[i] = buf[g - 1 - i];
        } else {
            ok = false;
            for (int i = m; i < k; ++i) w[i] = 0;
        }
    }
    uint32_t a = 0, c = 0, g_ = 0, t = 0;
    for (int i = 0; i < k; ++i) {
        uint32_t x = w[i];
        a |= (x & 1u) << i;
        c |= ((x >> 1) & 1u) << i;
        g_ |= ((x >> 2) & 1u) << i;
        t |= ((x >> 3) & 1u) << i;
    }
    out.a = a;
    out.c = c;
    out.g = g_;
    out.t = t;
    return ok;
}

// Terminal-gap patching of core:671-682 for a window that lies inside the row (p + k <= len), on bit-planes:
// the leading gap run (g cells) is replaced by the last g bases left of the window, the trailing run by the first
// g bases right of it — each only when the row holds that many bases there.  The flanks are found with clz / ffs
// on the "any base" word of each column word instead of walking cell by cell.
__device__ __forceinline__ void mpb_patch_edges(const uint32_t* __restrict__ pl, int64_t nsp, int64_t s, int len,
                                                int p, int k, uint32_t kmask, Win& w) {
    uint32_t gapv = ~(w.a | w.c | w.g | w.t) & kmask;
    if (gapv & 1u) {  // leading run
        const int g = __ffs(~gapv) - 1;  // < k because gapv != kmask
        uint32_t pa = 0, pc = 0, pg = 0, pt = 0;
        int got = 0;
        int j = (p - 1) >> 5;
        uint32_t below = (p & 31) ? ((1u << (p & 31)) - 1u) : 0xFFFFFFFFu;  // columns < p inside word j
        for (; j >= 0 && got < g; --j) {
            const uint4 q = mpb_word(pl, nsp, s, j);
            const uint32_t wa = q.x, wc = q.y, wg = q.z, wt = q.w;
            uint32_t any = (wa | wc | wg | wt) & below;
            below = 0xFFFFFFFFu;
            while (any && got < g) {
                const int b = 31 - __clz(any);
                any &= ~(1u << b);
                const int dst = g - 1 - got;  // nearest base goes right before the body
                pa |= ((wa >> b) & 1u) << dst;
                pc |= ((wc >> b) & 1u) << dst;
                pg |= ((wg >> b) & 1u) << dst;
                pt |= ((wt >> b) & 1u) << dst;
                ++got;
            }
        }
        if (p > 0 && got == g) {
            w.a |= pa;
            w.c |= pc;
            w.g |= pg;
            w.t |= pt;
            gapv = ~(w.a | w.c | w.g | w.t) & kmask;
        }
    }
    if ((gapv >> (k - 1)) & 1u) {  // trailing run (of the possibly updated window)
        const int g = __clz(~(gapv << (32 - k)));  // run of ones ending at bit k-1
        uint32_t pa = 0, pc = 0, pg = 0, pt = 0;
        int got = 0;
        const int c0 = p + k;
        const int jlast = (len - 1) >> 5;
        uint32_t above = ~((c0 & 31) ? ((1u << (c0 & 31)) - 1u) : 0u);  // columns >= c0 inside the first word
        for (int j = c0 >> 5; j <= jlast && got < g && c0 < len; ++j) {
            const uint4 q = mpb_word(pl, nsp, s, j);
            const uint32_t wa = q.x, wc = q.y, wg = q.z, wt = q.w;
            uint32_t any = (wa | wc | wg | wt) & above;  // cells >= len are stored as zero
            above = 0xFFFFFFFFu;
            while (any && got < g) {
                const int b = __ffs(any) - 1;
                any &= any - 1;
                const int dst = k - g + got;
                pa |= ((wa >> b) & 1u) << dst;
                pc |= ((wc >> b) & 1u) << dst;
                pg |= ((wg >> b) & 1u) << dst;
                pt |= ((wt >> b) & 1u) << dst;
                ++got;
            }
        }
        if (got == g) {
            w.a |= pa;
            w.c |= pc;
            w.g |= pg;
            w.t |= pt;
        }
    }
}

// Load the window starting at column p of sequence s.  Fast path: a funnel shift per plane.
__device__ __forceinline__ bool mpb_load_window(const uint32_t* __restrict__ pl, int64_t nsp, int64_t s, int len,
                                                int p, int k, uint32_t kmask, Win& w) {
    const uint4 w0 = mpb_word(pl, nsp, s, p >> 5);
    const uint4 w1 = mpb_word(pl, nsp, s, (p >> 5) + 1);
    const int sh = p & 31;
    w.a = __funnelshift_r(w0.x, w1.x, sh) & kmask;
    w.c = __funnelshift_r(w0.y, w1.y, sh) & kmask;
    w.g = __funnelshift_r(w0.z, w1.z, sh) & kmask;
    w.t = __funnelshift_r(w0.w, w1.w, sh) & kmask;
    uint32_t gapv = ~(w.a | w.c | w.g | w.t) & kmask;
    bool ok = true;
    if (p + k > len) {  // ragged row shorter than the window end: the generic cell-by-cell restatement
        Win t;
        ok = mpb_window_slow(pl, nsp, s, len, p, k, t);
        w.a = t.a;
        w.c = t.c;
        w.g = t.g;
        w.t = t.t;
        gapv = ~(w.a | w.c | w.g | w.t) & kmask;
    } else if (((gapv & 1u) | ((gapv >> (k - 1)) & 1u)) && gapv != kmask) {
        mpb_patch_edges(pl, nsp, s, len, p, k, kmask, w);
        gapv = ~(w.a | w.c | w.g | w.t) & kmask;
    }
    w.gapv = gapv;
    w.multi = mpb_multi(w.a, w.c, w.g, w.t);
    return ok;
}

// Number of expansions of a window holding IUPAC cells (saturates above MPB_MAX_EXP).
__device__ __forceinline__ uint32_t mpb_expansions(const Win& w) {
    uint32_t total = 1;
    uint32_t m = w.multi;
    while (m) {
        int i = __ffs(m) - 1;
        m &= m - 1;
        int code = ((w.a >> i) & 1u) | (((w.c >> i) & 1u) << 1) | (((w.g >> i) & 1u) << 2) | (((w.t >> i) & 1u) << 3);
        total *= c_fold[code];
        if (total > MPB_MAX_EXP) return MPB_MAX_EXP + 1;
    }
    return total;
}

// The e-th expansion (reference product order: leftmost position slowest) as one-hot planes.
__device__ __forceinline__ void mpb_expand(const Win& w, uint32_t e, uint32_t& a, uint32_t& c, uint32_t& g,
                                           uint32_t& t) {
    const uint32_t keep = ~w.multi;
    a = w.a & keep;
    c = w.c & keep;
    g = w.g & keep;
    t = w.t & keep;
    uint32_t m = w.multi;
    while (m) {
        int i = 31 - __clz(m);  // rightmost position varies fastest
        m &= ~(1u << i);
        int code = ((w.a >> i) & 1u) | (((w.c >> i) & 1u) << 1) | (((w.g >> i) & 1u) << 2) | (((w.t >> i) & 1u) << 3);
        uint32_t n = c_fold[code];
        uint32_t d = e % n;
        e /= n;
        uint32_t base = (c_order[code] >> (2 * d)) & 3u;
        uint32_t bit = 1u << i;
        a |= base == 0 ? bit : 0u;
        c |= base == 1 ? bit : 0u;
        g |= base == 2 ? bit : 0u;
        t |= base == 3 ? bit : 0u;
    }
}

// 64-bit key of a one-hot haplotype.  Gap-free: 2 bits per base, bit-sliced (low k bits = "C or T", next k
// bits = "G or T").  With gaps: MPB_KEY_BASE5 + sum d_i 5^i, d = 0..3 base, 4 gap.
__device__ __forceinline__ uint64_t mpb_key(uint32_t c, uint32_t g, uint32_t t, uint32_t gapv, int k) {
    if (gapv == 0) return (uint64_t)(c | t) | ((uint64_t)(g | t) << k);
    uint64_t x = 0;
    for (int i = 0; i < k; ++i) {
        uint32_t d = ((c >> i) & 1u) + 2u * ((g >> i) & 1u) + 3u * ((t >> i) & 1u) + 4u * ((gapv >> i) & 1u);
        x += (uint64_t)d * c_pow5[i];
    }
    return MPB_KEY_BASE5_D + x;
}

// digits (0..3 base, 4 gap) of a key -> planes
__device__ __forceinline__ void mpb_key_planes(uint64_t key, int k, uint32_t kmask, uint32_t& a, uint32_t& c,
                                               uint32_t& g, uint32_t& t, uint32_t& gapv) {
    if (key < MPB_KEY_BASE5_D) {
        uint32_t b0 = (uint32_t)key & kmask;
        uint32_t b1 = (uint32_t)(key >> k) & kmask;
        t = b0 & b1;
        c = b0 & ~b1;
        g = b1 & ~b0;
        a = ~(b0 | b1) & kmask;
        gapv = 0;
        return;
    }
    uint64_t x = key - MPB_KEY_BASE5_D;
    a = c = g = t = gapv = 0;
    for (int i = 0; i < k; ++i) {
        uint32_t d = (uint32_t)(x % 5ull);
        x /= 5ull;
        uint32_t bit = 1u << i;
        a |= d == 0 ? bit : 0u;
        c |= d == 1 ? bit : 0u;
        g |= d == 2 ? bit : 0u;
        t |= d == 3 ? bit : 0u;
        gapv |= d == 4 ? bit : 0u;
    }
}

__device__ __forceinline__ uint32_t mpb_hash(uint64_t key, int log2cap) {
    return (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> (64 - log2cap));
}

// open addressing, linear probing; count += add, first = min(first, ord).  The call that claims a slot appends it to
// the window's entry list (elist, n_new): the table readers walk that list instead of all slots.
__device__ __forceinline__ void mpb_table_add(uint64_t* __restrict__ keys, uint32_t* __restrict__ cnt,
                                              uint64_t* __restrict__ first, int log2cap, uint64_t key, uint32_t add,
                                              uint64_t ord, int* err, unsigned long long* n_new,
                                              uint32_t* __restrict__ elist) {
    const uint32_t mask = (1u << log2cap) - 1u;
    const uint32_t last_probe = mask < 8191u ? mask : 8191u;  // a run this long means the table is as good as full
    uint32_t h = mpb_hash(key, log2cap);
    for (uint32_t probe = 0; probe <= last_probe; ++probe) {
        uint64_t cur = *((volatile uint64_t*)&keys[h]);
        if (cur == MPB_KEY_EMPTY_D) {
            cur = atomicCAS((unsigned long long*)&keys[h], (unsigned long long)MPB_KEY_EMPTY_D,
                            (unsigned long long)key);
            if (cur == MPB_KEY_EMPTY_D) {
                cur = key;
                const unsigned long long idx = atomicAdd(n_new, 1ull);  // this call claimed the slot
                elist[idx] = h;
            }
        }
        if (cur == key) {
            atomicAdd(&cnt[h], add);
            // `first` only ever decreases: a row that is not earlier than the value already there needs no atomic
            if (*((volatile uint64_t*)&first[h]) > ord) atomicMin((unsigned long long*)&first[h], (unsigned long long)ord);
            return;
        }
        h = (h + 1) & mask;
    }
    atomicOr(err, MPB_ERR_TABLE_FULL);
}
