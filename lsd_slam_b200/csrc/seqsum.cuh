// seqsum.cuh -- the reference's SEQUENTIAL fp32 sum, reproduced bit for bit by a parallel kernel.
//
// DepthMap::createKeyFrame rescales the new keyframe's map by numIdepth / sumIdepth, where sumIdepth is a plain
// `float += idepth_smoothed` over the valid hypotheses in raster order (DepthMap.cpp:1286-1294).  Its rounding errors
// (~1e-5 relative over 1.2e5 terms) enter every hypothesis of the new keyframe, so a tree or double-precision sum makes the
// whole map differ from the reference in the 5th digit.  This file computes the SAME float the sequential loop produces.
//
// How.  While the running sum s stays inside one binade [2^k, 2^(k+1)), s = S * u with u = 2^(k-23) and S a 24-bit integer,
// and IEEE round-to-nearest-even gives  fl(s + x) = u * RNE(S + x/u):  writing x/u = n + f,
//      S' = S + n + [f > 1/2] + [f == 1/2 and (S + n) odd].
// For x > 0 that is an integer map  S -> S + (S even ? d0 : d1)  with (d0, d1) depending on x and k only; such maps are closed
// under composition, and composition is associative -- so inside a binade the sequential sum is a SCAN.  Pass 1 (k_seqsum_table,
// the whole GPU) composes the maps of every run of 256 pixels for each binade k = 0..23.  Pass 2 (k_seqsum_walk, one warp) scans
// 32 runs at a time with the table of the current binade, stops at the first run in which S would reach 2^24 (the sum leaves the
// binade: a few dozen times per image since the terms are positive) and resolves that run 32 pixels at a time with maps built on
// the fly, performing the one addition that crosses the binade with a real float add.  Anything outside the model (x <= 0, NaN,
// s not a positive normal number) is added with a real float add, one element at a time, so the result is the sequential sum
// for ANY input; the fast path only needs the positive terms the mapper produces.
#pragma once
#include "internal.cuh"      // SEQ_NBIN, SEQ_RUN

#define SEQ_SAT (1 << 28)    // saturation of the increments: > 2^24, so "reached 2^24" survives, and below 2^24 nothing saturates

struct SeqMap { int d0, d1; };   // S -> S + (S even ? d0 : d1)

__host__ __device__ __forceinline__ SeqMap seqIdentity() { SeqMap m; m.d0 = 0; m.d1 = 0; return m; }

// f first, then g
__host__ __device__ __forceinline__ SeqMap seqCompose(SeqMap f, SeqMap g)
{
    SeqMap r;
    int a = f.d0 + ((f.d0 & 1) ? g.d1 : g.d0);            // S even -> S + f.d0 has the parity of f.d0
    int b = f.d1 + ((f.d1 & 1) ? g.d0 : g.d1);            // S odd  -> S + f.d1 is odd iff f.d1 is even
    r.d0 = a < SEQ_SAT ? a : SEQ_SAT;
    r.d1 = b < SEQ_SAT ? b : SEQ_SAT;
    return r;
}

// the map of one term x > 0 (finite) while the sum is in binade k
__host__ __device__ __forceinline__ SeqMap seqElement(unsigned int xbits, int k)
{
    int e = (int)((xbits >> 23) & 0xffu);
    unsigned int m = xbits & 0x7fffffu;
    if (e) m |= 0x800000u; else e = 1;                    // denormal terms: no implicit one, exponent of the smallest normal
    const int sh = (e - 127) - k;                         // x / u = m * 2^sh
    SeqMap r;
    if (sh >= 0) {
        int n = sh >= 5 ? SEQ_SAT : (int)(m << sh);       // m < 2^24: m << 4 < 2^28
        if (n > SEQ_SAT) n = SEQ_SAT;
        r.d0 = n; r.d1 = n;
        return r;
    }
    const int rs = -sh;
    if (rs > 25) { r.d0 = 0; r.d1 = 0; return r; }        // x < u/2: absorbed (f < 1/2, n = 0)
    const unsigned int n = rs >= 32 ? 0u : (m >> rs);
    const unsigned int rem = m & ((1u << rs) - 1u);
    const unsigned int half = 1u << (rs - 1);
    const int up = rem > half;
    const int tie = rem == half;
    r.d0 = (int)n + up + (tie & (int)(n & 1u));           // S even: S + n odd iff n odd
    r.d1 = (int)n + up + (tie & (int)(~n & 1u));          // S odd : S + n odd iff n even
    return r;
}

__host__ __device__ __forceinline__ bool seqIsFastTerm(unsigned int xbits)
{   // x > 0 and finite (denormals included)
    return (xbits >> 31) == 0 && xbits != 0 && (xbits >> 23) != 0xffu;
}

#ifdef __CUDACC__
__device__ __forceinline__ SeqMap seqShflDown(SeqMap m, int o)
{
    SeqMap r;
    r.d0 = __shfl_down_sync(0xffffffffu, m.d0, o);
    r.d1 = __shfl_down_sync(0xffffffffu, m.d1, o);
    return r;
}
__device__ __forceinline__ SeqMap seqShflUp(SeqMap m, int o)
{
    SeqMap r;
    r.d0 = __shfl_up_sync(0xffffffffu, m.d0, o);
    r.d1 = __shfl_up_sync(0xffffffffu, m.d1, o);
    return r;
}

// pass 1: one warp per run of 256 pixels (lane owns 8 consecutive ones).  table[k * nRuns + run] = composed map of the run in
// binade k; flags[run] = the run holds a valid term outside the fast path; counts[run] = its valid pixels.
__global__ void __launch_bounds__(256) k_seqsum_table(const float4* __restrict__ hf, const int4* __restrict__ hi, int n, int nRuns,
                                                      int2* __restrict__ table, unsigned char* __restrict__ flags, int* __restrict__ counts)
{
    const int lane = threadIdx.x & 31;
    const int run = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (run >= nRuns) return;
    unsigned int xb[8];
    unsigned int validMask = 0;
    bool special = false;
    const int base = run * SEQ_RUN + lane * 8;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int i = base + j;
        xb[j] = 0;
        if (i < n && hi[i].x) {
            xb[j] = __float_as_uint(hf[i].z);
            if (seqIsFastTerm(xb[j])) validMask |= 1u << j; else special = true;
        }
    }
    int cnt = __popc(validMask) + 0;
    if (special) {   // count the special ones too (they are valid hypotheses)
        cnt = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) { const int i = base + j; if (i < n && hi[i].x) cnt++; }
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    const bool anySpecial = __any_sync(0xffffffffu, special);
    if (lane == 0) { flags[run] = anySpecial ? 1 : 0; counts[run] = cnt; }
#pragma unroll 1
    for (int k = 0; k < SEQ_NBIN; k++) {
        SeqMap m = seqIdentity();
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (validMask & (1u << j)) m = seqCompose(m, seqElement(xb[j], k));
        for (int o = 1; o < 32; o <<= 1) {                 // ordered reduction: lane l ends with the map of lanes l .. l+2o-1
            SeqMap other = seqShflDown(m, o);
            if (lane + o < 32) m = seqCompose(m, other);
        }
        if (lane == 0) table[(size_t)k * nRuns + run] = make_int2(m.d0, m.d1);
    }
}

__device__ __forceinline__ bool seqSumIsFast(float s)
{   // positive normal finite
    const unsigned int b = __float_as_uint(s);
    const unsigned int e = (b >> 23) & 0xffu;
    return (b >> 31) == 0 && e != 0 && e != 0xffu;
}

// one warp advances the sum over up to 32 items given as maps of the CURRENT binade (inclusive scan), returns the index of the
// first item it could not absorb (32 = all absorbed) and leaves s = the sum before that item
__device__ __forceinline__ int seqAdvance(float& s, SeqMap m, bool mustStop, int lane)
{
    const unsigned int sb = __float_as_uint(s);
    const int S = (int)((sb & 0x7fffffu) | 0x800000u);
    for (int o = 1; o < 32; o <<= 1) {
        SeqMap prev = seqShflUp(m, o);
        if (lane >= o) m = seqCompose(prev, m);
    }
    const int Sout = S + ((S & 1) ? m.d1 : m.d0);
    const unsigned int stop = __ballot_sync(0xffffffffu, mustStop || Sout >= (1 << 24));
    const int first = stop ? (__ffs(stop) - 1) : 32;
    const int src = first == 0 ? 0 : first - 1;
    int Sprev = __shfl_sync(0xffffffffu, Sout, src);
    if (first == 0) Sprev = S;
    s = __uint_as_float((sb & 0x7f800000u) | ((unsigned int)Sprev & 0x7fffffu));
    return first;
}

// the 256 pixels of one run, 32 at a time, maps built for whatever binade the sum is in
__device__ __forceinline__ void seqWalkRun(float& s, const float4* __restrict__ hf, const int4* __restrict__ hi, int n, int run, int lane)
{
    float xv[8];
    bool vv[8];
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int i = run * SEQ_RUN + r * 32 + lane;
        vv[r] = i < n && hi[i].x != 0;
        xv[r] = vv[r] ? hf[i].z : 0.0f;
    }
#pragma unroll 1
    for (int r = 0; r < 8; r++) {
        const float x = xv[r];
        const bool v = vv[r];
        unsigned int remaining = __ballot_sync(0xffffffffu, v);
        while (remaining) {
            const int firstLane = __ffs(remaining) - 1;
            if (!seqSumIsFast(s)) {                        // s is 0, negative, denormal, inf or NaN: one real addition
                s = __fadd_rn(s, __shfl_sync(0xffffffffu, x, firstLane));
                remaining &= ~(1u << firstLane);
                continue;
            }
            const int k = (int)((__float_as_uint(s) >> 23) & 0xffu) - 127;
            const bool mine = (remaining >> lane) & 1u;
            const unsigned int xb = __float_as_uint(x);
            const bool fast = seqIsFastTerm(xb);
            SeqMap m = (mine && fast) ? seqElement(xb, k) : seqIdentity();
            const int first = seqAdvance(s, m, mine && !fast, lane);
            if (first == 32) break;
            s = __fadd_rn(s, __shfl_sync(0xffffffffu, x, first));       // the addition that leaves the binade (or a special term)
            remaining &= ~((2u << first) - 1u);
        }
    }
}

// pass 2: out[0] = the sequential float sum, out[1] = number of valid hypotheses, out[2] = (float)count / sum as in :1294
__global__ void __launch_bounds__(32) k_seqsum_walk(const float4* __restrict__ hf, const int4* __restrict__ hi, int n, int nRuns,
                                                    const int2* __restrict__ table, const unsigned char* __restrict__ flags,
                                                    const int* __restrict__ counts, double* __restrict__ out)
{
    const int lane = threadIdx.x;
    int cnt = 0;
    for (int r = lane; r < nRuns; r += 32) cnt += counts[r];
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    float s = 0.0f;
    int run = 0;
    while (run < nRuns) {
        const int k = (int)((__float_as_uint(s) >> 23) & 0xffu) - 127;
        if (!seqSumIsFast(s) || k < 0 || k >= SEQ_NBIN) { seqWalkRun(s, hf, hi, n, run, lane); run++; continue; }
        const int r = run + lane;
        SeqMap m = seqIdentity();
        bool special = false;
        if (r < nRuns) {
            const int2 t = __ldg(table + (size_t)k * nRuns + r);
            m.d0 = t.x; m.d1 = t.y;
            special = flags[r] != 0;
        }
        const int first = seqAdvance(s, m, special, lane);
        run += first;
        if (first < 32) { seqWalkRun(s, hf, hi, n, run, lane); run++; }
    }
    if (lane == 0) {
        out[0] = (double)s;
        out[1] = (double)cnt;
        out[2] = (double)__fdiv_rn((float)cnt, s);
    }
}
#endif
