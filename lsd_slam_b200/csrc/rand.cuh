// rand.cuh -- glibc's random() (stdlib/random_r.c), which rand() calls, as a generator that can jump to any draw: the stream
// DepthMap::initializeRandomly (DepthEstimation/DepthMap.cpp:883-916) draws its hypotheses from.  Host and device share it.
//
// TYPE_0 is the LCG s' = (s * 1103515245 + 12345) & 0x7fffffff; the draw is s'.  TYPE_1..TYPE_4 are additive lagged-Fibonacci
// generators over Z/2^32 with (deg, sep) = (7, 3), (15, 1), (31, 3), (63, 1): the table word at the front pointer gets the word
// at the rear pointer added, and the draw is the new word >> 1.  Written as one sequence v, v[i] = v[i - deg] + v[i - sep], and
// the state before draw k is the WINDOW W[m] = v[k - deg + m], m < deg.  In glibc's table with rear index `rear` (the rear
// pointer) the window starts at the front pointer: W[m] = table[(rear + sep + m) % deg].
//
// Jump-ahead: with P(x) = x^deg - x^(deg-sep) - 1 and p(x) = x^t mod P = sum_j p[j] x^j, every solution of the recurrence has
// v[i + t] = sum_j p[j] v[i + j], so the window t draws later is W'[m] = sum_j p[j] ext[m + j], where ext = the window followed by
// its next deg-1 values.  All of it is uint32 arithmetic with wrap-around, exact like glibc's.  The tables below hold
// x^(2^b) mod P (the jumps) and x^(deg+j) mod P (v[k + j] = sum_m gen[j][m] W[m]: the next draws straight from a window).
//
// Table sizes (internal.cuh): RND_ROW words per polynomial or window (deg <= 63, zero-padded); per type RND_POW_ROWS jump rows
// (any jump below 2^63 draws) and RND_GEN_ROWS draw rows.
#pragma once
#include "internal.cuh"

struct RndKind { int deg, sep; };

// random_poly_info, stdlib/random_r.c: degrees { 0, 7, 15, 31, 63 }, separations { 0, 3, 1, 3, 1 }
__host__ __device__ inline RndKind rndKind(int type)
{
    switch (type) {
    case 1: return { 7, 3 };
    case 2: return { 15, 1 };
    case 3: return { 31, 3 };
    case 4: return { 63, 1 };
    default: return { 0, 0 };
    }
}
// words of the window: deg, and the LCG's single state word
__host__ __device__ inline int rndWindowLen(int type) { return type == 0 ? 1 : rndKind(type).deg; }

// sum of a[i] * b[i] for i = start, start + stride, ... < n, mod 2^32
__host__ __device__ inline uint32_t rndDot(const uint32_t* a, const uint32_t* b, int n, int start, int stride)
{
    uint32_t s = 0;
    for (int i = start; i < n; i += stride) s += a[i] * b[i];
    return s;
}

// the LCG's t-step map s -> A s + C (mod 2^32; the mask of every step commutes with it), by squaring
__host__ __device__ inline void rndLcgJump(uint64_t t, uint32_t& A, uint32_t& C)
{
    uint32_t a = 1103515245u, c = 12345u;
    A = 1u; C = 0u;
    while (t) {
        if (t & 1) { C = a * C + c; A = a * A; }
        c = a * c + c; a = a * a;
        t >>= 1;
    }
}
__host__ __device__ inline uint32_t rndLcgAt(uint32_t s0, uint64_t t)
{
    uint32_t A, C;
    rndLcgJump(t, A, C);
    return (A * s0 + C) & 0x7fffffffu;
}

// what rand() returns for sequence value v
__host__ __device__ inline int32_t rndOutput(int type, uint32_t v) { return (int32_t)(type == 0 ? v : v >> 1); }

// DepthMap.cpp:898: 0.5f + 1.0f * ((rand() % 100001) / 100000.0f), fp32 with round-to-nearest at every step
__device__ __forceinline__ float rndIdepth(int32_t r)
{
    return __fadd_rn(0.5f, __fmul_rn(1.0f, __fdiv_rn((float)(r % 100001), 100000.0f)));
}

// ---- host side: the tables, srandom_r and random_r ------------------------------------------------------------------------
// p <- p * q mod P (deg coefficients each)
static inline void rndPolyMulMod(const uint32_t* p, const uint32_t* q, uint32_t* out, RndKind k)
{
    uint32_t c[2 * RND_ROW] = {};
    for (int i = 0; i < k.deg; i++)
        for (int j = 0; j < k.deg; j++) c[i + j] += p[i] * q[j];
    for (int i = 2 * k.deg - 2; i >= k.deg; i--) {           // x^i = x^(i-sep) + x^(i-deg)
        c[i - k.sep] += c[i];
        c[i - k.deg] += c[i];
    }
    for (int i = 0; i < RND_ROW; i++) out[i] = i < k.deg ? c[i] : 0u;
}

// per type: RND_POW_ROWS rows x^(2^b) mod P, then RND_GEN_ROWS rows x^(deg+j) mod P (all zero for TYPE_0)
struct RndTables {
    uint32_t w[RND_TYPES][RND_TYPE_WORDS];
    RndTables()
    {
        for (int t = 0; t < RND_TYPES; t++) {
            uint32_t* tab = w[t];
            for (int i = 0; i < RND_TYPE_WORDS; i++) tab[i] = 0;
            const RndKind k = rndKind(t);
            if (!k.deg) continue;
            tab[1] = 1;                                       // x
            for (int b = 1; b < RND_POW_ROWS; b++) rndPolyMulMod(tab + (b - 1) * RND_ROW, tab + (b - 1) * RND_ROW, tab + b * RND_ROW, k);
            uint32_t* gen = tab + RND_POW_ROWS * RND_ROW;
            gen[k.deg - k.sep] = 1; gen[0] = 1;               // x^deg = x^(deg-sep) + 1
            for (int j = 1; j < RND_GEN_ROWS; j++) {          // times x
                const uint32_t* p = gen + (j - 1) * RND_ROW;
                uint32_t* q = gen + j * RND_ROW;
                const uint32_t top = p[k.deg - 1];
                for (int i = k.deg - 1; i > 0; i--) q[i] = p[i - 1];
                q[0] = top;
                q[k.deg - k.sep] += top;
            }
        }
    }
};
static inline const RndTables& rndTables()
{
    static const RndTables* t = new RndTables();             // built once, on first use
    return *t;
}

// glibc table + rear <-> window
static inline void rndTableToWindow(int type, int rear, const uint32_t* table, uint32_t* W)
{
    const RndKind k = rndKind(type);
    if (type == 0) { W[0] = table[0]; return; }
    for (int m = 0; m < k.deg; m++) W[m] = table[(rear + k.sep + m) % k.deg];
}
static inline void rndWindowToTable(int type, int rear, const uint32_t* W, uint32_t* table)
{
    const RndKind k = rndKind(type);
    if (type == 0) { table[0] = W[0]; return; }
    for (int m = 0; m < k.deg; m++) table[(rear + k.sep + m) % k.deg] = W[m];
}

// the window n draws later (TYPE_1..4): one jump per set bit of n
static inline void rndJumpWindow(int type, uint32_t* W, uint64_t n)
{
    const RndKind k = rndKind(type);
    const uint32_t* tab = rndTables().w[type];
    for (int b = 0; n; b++, n >>= 1) {
        if (!(n & 1)) continue;
        uint32_t ext[2 * RND_ROW];
        for (int i = 0; i < k.deg; i++) ext[i] = W[i];
        for (int i = k.deg; i < 2 * k.deg - 1; i++) ext[i] = ext[i - k.deg] + ext[i - k.sep];
        for (int m = 0; m < k.deg; m++) W[m] = rndDot(tab + b * RND_ROW, ext + m, k.deg, 0, 1);
    }
}
