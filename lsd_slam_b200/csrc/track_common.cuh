// track_common.cuh -- what the three device trackers share: the SE3 tracker (track_persistent.cuh), permaRef tracking
// (perma.cuh) and Sim3 tracking (sim3.cuh).  Device code only, no kernel: the parameter and result blocks, the LM state machine
// of SE3Tracker::trackFrame (Tracking/SE3Tracker.cpp:280-486) with its solves, the multi-value warp reductions, and the layouts
// of the batch descriptors and results the context's arena holds.
#pragma once
#include "internal.cuh"
#include "track.cuh"

#define TP_THREADS 512
#define TP_WARPS (TP_THREADS / 32)
#define TP_MAXGRID 160               // combine code is unrolled for <= 160 CTAs (H100 SXM: 132 SMs)
#define TP_SYNC_WORDS 4096           // ctx->trkSync: word 0 = arrival counter of the grid barrier
#define TP_MAX_RANKS 8               // GPUs one stream's tracking can be sharded over (peer exchange, see gridExchangeRanks)
#define TP_XCHG_OFFSET 1024          // word offset of the cross-GPU exchange rows: [TP_MAX_RANKS][64] slots of {value, tag} (8 B each)
#define TP_DONE_OFFSET 3072          // word offset of the per-peer "my writes into your memory are complete" slots (8 B each)
#define TP_TAIL_OFFSET 3200          // word: arrival counter of the end-of-kernel barrier of a sharded launch
#define TP_KMAX 3                    // poses per pass: the try + up to two speculative successors
#define TP_ROW 64                    // floats per exchange row (256 B, one row per CTA; EV_NCHX = 56 used)
#define TP_MAX_GROUP 8               // streams one group launch can track (lsdgpu_track_and_map_group)

struct TrackLevelParams {
    const float* kfIdepth;
    const float* kfVar;
    const float* kfColor;
    const float4* frameGrad;
    int w, h;
    float fx, fy, cx, cy, fxi, fyi, cxi, cyi;
    // Only INTERIOR pixels can be points (TrackingReference.cpp:128-129 scans 1..w-2 x 1..h-2); they are numbered row by row,
    // j = (x-1) + (y-1)*iw, and cut into chunks of 32 consecutive j (chunk c -> CTA c % gridDim, warp slot c / gridDim).
    // At 640x480 level 1 has 318*238 = 75 684 interior pixels = 2 366 chunks over 132 CTAs x 16 warps: one or two chunks per warp.
    int iw, nInt, nChunks;
};

struct TrackParams {
    TrackLevelParams lvl[LSD_LEVELS];
    uint8_t* goodMask;               // level-1 mask of the tracked frame
    int maskFresh;                   // 1: initialise the mask to true first (Frame.h:433)
    int maskBytes;
    int W, H;                        // tracker construction size (diverge test uses width>>lvl, SE3Tracker.cpp:324)
    float initRefToFrame[7];         // frameToReference_initialEstimate.inverse().cast<float>(), :306
    lsdgpu_track_settings st;
    EvalConsts C;
    int useAffine;
    float* partials;                 // [2][gridDim][TP_ROW]
    unsigned int* sync;              // word 0: arrival counter of the grid barrier (monotonic, never reset)
    unsigned int barrierBase;        // arrivals counted by earlier launches
    int debug;                       // 1: also write the per-CTA cycle table
    unsigned int launchSeq;          // value the kernel stores in TrackState::doneSeq when the result block is complete
    int minLevel;                    // last level of the coarse-to-fine loop (1 for trackFrame, 4 for permaRef tracking)
    int kmax;                        // candidate poses per pass (TP_KMAX for trackFrame, 1 = no speculation for permaRef tracking)
    // one stream sharded over nRanks GPUs (BASELINE config 5): this GPU evaluates every nRanks-th chunk; the per-pass sums and the
    // level-1 mask are exchanged through peer-mapped memory inside the kernel (no host, no NCCL call on the path)
    int nRanks, rank;
    unsigned int* peerSync[TP_MAX_RANKS];     // each rank's `sync` block as mapped into THIS process (own entry = sync)
    uint8_t* peerMask[TP_MAX_RANKS];          // the tracked frame's level-1 mask on each rank
    unsigned int tailBase;                    // arrivals already counted on the tail barrier
    // level-1 good flags of the last candidate of a pass (the context's plane; goodMask holds candidate 0's), committed at the end
    // of the launch if that candidate was the last pose the reference evaluates
    uint8_t* lastMask;
};

// what the kernel hands back (block 0 writes it)
struct TrackState {
    float refToFrame[7];
    float pointUsage, goodCount, badCount, meanRes, lastResidual;
    float affine_a, affine_b;
    int diverged;
    int numCalcResidualCalls[LSD_LEVELS];
    int numCalcWarpUpdateCalls[LSD_LEVELS];
    int evalsAtLevel[LSD_LEVELS];    // passes per level
    float pointsAtLevel[LSD_LEVELS]; // numData[level]: valid points of the keyframe on each tracked level (CH_REFNUM)
    int posesEvaluated;              // poses evaluated including the speculative ones (>= sum of numCalcResidualCalls)
    int totalEvals;                  // passes (= grid barriers) of this launch
    volatile unsigned int doneSeq;   // written last (after a system-wide fence): the host polls it instead of a stream sync
    long long cyc[6];                // block-0 cycle breakdown: points, CTA reduce, barrier, combine, serial LM, total
    long long cycBlk[TP_MAXGRID][6];   // the same per CTA (debug); the last row holds warp 0's cycles
};

// ---- several streams in one launch (k_track_persistent_group) ------------------------------------------------------------------
// The launch is cut into n segments of Gs = floor(trackGrid / n) CTAs; segment s tracks stream s with its own parameters, partial
// rows, barrier counter and result block.  A segment keeps the single-stream launch's VIRTUAL grid of Gv = trackGrid CTAs: its
// physical CTA b stands in for the virtual CTAs b, b + Gs, ... < Gv one after the other, evaluating exactly the chunks, with the
// same warp / lane mapping, and writing exactly the row that virtual CTA writes in a single-stream launch.  The combine then adds
// the same Gv rows in the same order, so every sum, every LM decision and every result is bit-identical to k_track_persistent's.
// A native grid of Gs CTAs would deal the chunks out differently and change the fp32 summation order.
struct TrackGroupSeg {
    TrackParams p;                   // the stream's parameters (nRanks == 1, debug == 0)
    TrackState* out;                 // its context's mapped result block
};
enum { ACT_CONTINUE = 0, ACT_LEVEL_DONE = 1, ACT_DIVERGED = 2 };

// one candidate pose of a chain
struct Cand {
    lsd::SE3<float> T;
    float inc[6];
    float lambda, incSq;
};

struct LMShared {
    float sums[EV_NCHX];             // [0, EV_NCH): candidate 0; [EV_NCH, EV_NCHX): extension block of the other candidates
    EvalPose pose[TP_KMAX];          // poses of the next pass
    int nPose;                       // how many of them
    int action;
    int lvl;                         // level of the next pass
    Cand cand[TP_KMAX];
};

__device__ __forceinline__ void setEvalPose(EvalPose& P, const lsd::SE3<float>& T, float a, float b)
{
    lsd::quatToMatrix(T.q, P.R);
    P.t[0] = T.t[0]; P.t[1] = T.t[1]; P.t[2] = T.t[2];
    P.a = a; P.b = b;
}

// ---- multi-value warp reduction -------------------------------------------------------------------------
// K values per lane (K a power of two <= 32) are reduced across the warp with K-1 (+ log2(32/K)) shuffles
// instead of 5K: at every step the lanes of a pair exchange HALF of their values.  On return v[0] holds the
// warp total of channel  chan = sum over used masks of (lane & mask ? half : 0)  (for K = 32: chan == lane).
// Fixed exchange pattern => bit-identical results wherever the same data is reduced.
// Each stage is its own instantiation (HALF a compile-time constant), so that every v[i + HALF] is a fixed register: written as one
// loop over `half >>= 1` the array lived in local memory, a load and a store per element and stage (the CTA reduce was the largest
// phase of the tracker's pass, DESIGN §6).  The lane's pick between the two values is a bit-mask select.
template <int HALF, int K, typename T>
__device__ __forceinline__ void warpReduceStage(T (&v)[K], int lane, int mask)
{
    const unsigned int up = (lane & mask) ? 0xffffffffu : 0u;
#pragma unroll
    for (int i = 0; i < HALF; i++) {
        const unsigned int lo = __float_as_uint(v[i]), hi = __float_as_uint(v[i + HALF]);
        const T keep = __uint_as_float((lo & ~up) | (hi & up));              // (lane & mask) ? v[i + HALF] : v[i]
        const T send = __uint_as_float((hi & ~up) | (lo & up));              // (lane & mask) ? v[i] : v[i + HALF]
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, mask);
    }
    if constexpr (HALF > 1) warpReduceStage<HALF / 2>(v, lane, mask >> 1);
}
template <int K, typename T>
__device__ __forceinline__ void warpReduceMulti(T (&v)[K], int lane)
{
    static_assert(K >= 2 && K <= 32 && (K & (K - 1)) == 0, "K is a power of two in [2, 32]");
    warpReduceStage<K / 2>(v, lane, 16);
#pragma unroll
    for (int mask = 16 / (K / 2) / 2; mask >= 1; mask >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], mask);
}
// channel held in v[0] by `lane` after warpReduceMulti<K>
template <int K> __device__ __forceinline__ int warpReduceChannel(int lane)
{
    int c = 0, mask = 16;
#pragma unroll
    for (int half = K / 2; half >= 1; half >>= 1, mask >>= 1)
        if (lane & mask) c += half;
    return c;
}


// all channels of a thread's accumulators -> per-warp totals in smRow: EV_NCH (= 32 + 8; 39 shuffles) and, when the pass
// carries more than one candidate, the 16 extension channels (16 more)
__device__ __forceinline__ void warpReduceAcc(PointAcc& acc, int lane, float* smRow)
{
    float a32[32], a8[8];
#pragma unroll
    for (int i = 0; i < 32; i++) a32[i] = acc.v[i];
#pragma unroll
    for (int i = 0; i < 8; i++) a8[i] = acc.v[32 + i];
    warpReduceMulti<32>(a32, lane);
    warpReduceMulti<8>(a8, lane);
    smRow[lane] = a32[0];
    if ((lane & 3) == 0) smRow[32 + warpReduceChannel<8>(lane)] = a8[0];
}
__device__ __forceinline__ void warpReduceExt(float (&x)[EV_NX], int lane, float* smRow)
{
    warpReduceMulti<EV_NX>(x, lane);
    if ((lane & 1) == 0) smRow[EV_NCH + warpReduceChannel<EV_NX>(lane)] = x[0];
}

// Fully unrolled, register-resident LDL^T without pivoting for the damped N x N normal equations (6x6 SE3, 7x7 Sim3); false if
// a pivot is not strictly positive (the caller then falls back to the pivoted routine of hostmath.h, which is what Eigen's
// ldlt() does).
template <int N> __device__ __forceinline__ bool ldltSolveFast(const float* A, const float* b, float* x)
{
    float Lm[N][N], D[N];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < N; j++) {
        float d = A[j * N + j];
#pragma unroll
        for (int k = 0; k < j; k++) d -= Lm[j][k] * Lm[j][k] * D[k];
        D[j] = d;
        ok = ok && (d > 0.f);
        const float inv = 1.0f / d;
#pragma unroll
        for (int i = j + 1; i < N; i++) {
            float v = A[i * N + j];
#pragma unroll
            for (int k = 0; k < j; k++) v -= Lm[i][k] * Lm[j][k] * D[k];
            Lm[i][j] = v * inv;
        }
    }
    float y[N];
#pragma unroll
    for (int i = 0; i < N; i++) {
        float s = b[i];
#pragma unroll
        for (int k = 0; k < i; k++) s -= Lm[i][k] * y[k];
        y[i] = s;
    }
#pragma unroll
    for (int i = 0; i < N; i++) y[i] = y[i] / D[i];
#pragma unroll
    for (int i = N - 1; i >= 0; i--) {
        float s = y[i];
#pragma unroll
        for (int k = i + 1; k < N; k++) s -= Lm[k][i] * x[k];
        x[i] = s;
    }
    return ok;
}

// exp(inc) * T on the device, latency-trimmed: one sincosf (half angle; sin/cos of the full angle by the
// double-angle identities), reciprocal-sqrt normalisations.  Same algebra as lsd::se3Exp / se3Mul (hostmath.h,
// se3.hpp:406-428, 239-259); results agree to ~1e-7 relative.
__device__ __forceinline__ lsd::SE3<float> se3ExpMulFast(const float* a, const lsd::SE3<float>& T)
{
    const float wx = a[3], wy = a[4], wz = a[5];
    const float theta_sq = wx * wx + wy * wy + wz * wz;
    float imag, real, c1, c2;
    if (theta_sq < 1e-10f) {
        const float theta_po4 = theta_sq * theta_sq;
        imag = 0.5f - (1.0f / 48.0f) * theta_sq + (1.0f / 3840.0f) * theta_po4;
        real = 1.0f - 0.5f * theta_sq + (1.0f / 384.0f) * theta_po4;
        c1 = 0.5f; c2 = 1.0f / 6.0f;                       // V = I + Omega/2 + Omega^2/6 (theta -> 0)
    } else {
        const float inv_theta = rsqrtf(theta_sq);
        const float theta = theta_sq * inv_theta;
        float sh_, ch_;
        sincosf(0.5f * theta, &sh_, &ch_);
        imag = sh_ * inv_theta;
        real = ch_;
        const float inv_sq = inv_theta * inv_theta;
        c1 = 2.0f * sh_ * sh_ * inv_sq;                     // (1 - cos theta) / theta^2
        c2 = (theta - 2.0f * sh_ * ch_) * inv_sq * inv_theta;   // (theta - sin theta) / theta^3
    }
    float q[4] = { imag * wx, imag * wy, imag * wz, real };
    {
        const float n = rsqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        q[0] *= n; q[1] *= n; q[2] *= n; q[3] *= n;
    }
    // V * upsilon with V = I + c1*Omega + c2*Omega^2 :  Omega u = w x u,  Omega^2 u = w x (w x u)
    const float ux = a[0], uy = a[1], uz = a[2];
    const float k1x = wy * uz - wz * uy, k1y = wz * ux - wx * uz, k1z = wx * uy - wy * ux;
    const float k2x = wy * k1z - wz * k1y, k2y = wz * k1x - wx * k1z, k2z = wx * k1y - wy * k1x;
    const float tx = ux + c1 * k1x + c2 * k2x, ty = uy + c1 * k1y + c2 * k2y, tz = uz + c1 * k1z + c2 * k2z;
    // (q, t) * T
    lsd::SE3<float> r;
    float rt[3];
    lsd::quatRotate(q, T.t, rt);
    lsd::quatMul(q, T.q, r.q);
    {
        const float n = rsqrtf(r.q[0] * r.q[0] + r.q[1] * r.q[1] + r.q[2] * r.q[2] + r.q[3] * r.q[3]);
        r.q[0] *= n; r.q[1] *= n; r.q[2] *= n; r.q[3] *= n;
    }
    r.t[0] = tx + rt[0]; r.t[1] = ty + rt[1]; r.t[2] = tz + rt[2];
    return r;
}

// LM state of SE3Tracker::trackFrame; lives in shared memory, touched by warp 0 only (keeps it out of the
// register budget of the point loop)
struct LMState {
    lsd::SE3<float> refToFrame, cand;
    float affine_a, affine_b, lastErr, last_residual, LM_lambda;
    float inc[6];
    float lsq[27];                   // accepted normal equations, RAW sums: 21 upper-triangle A + 6 (sum J r w)
    int nRes[LSD_LEVELS], nUpd[LSD_LEVELS], nEval[LSD_LEVELS];
    float nPts[LSD_LEVELS];
    int lvl, iteration, phase, incTry, diverged;
    int chainBase;                   // lm.incTry when the chain of the pass in flight was built
    int statsFrom;                   // where the statistics of the last evaluated pose are: 0 = main block, 1 = extension block
    int commitLast;                  // 1: the good-mask of the last evaluated pose is in TrackParams::lastMask, not yet in the mask
    int posesEvaluated;
    long long dbg[4];                // warp-0 cycles: decisions, chain building
};
enum { PH_INIT = 0, PH_TRY = 1, PH_REEVAL = 2 };

// affine lighting estimate of the last evaluation, SE3Tracker.cpp:1023-1024
__device__ __forceinline__ void affineFromSums(const float* s, float& a, float& b)
{
    const float sxx = s[CH_SXX], syy = s[CH_SYY], sx = s[CH_SX], sy = s[CH_SY], sw = s[CH_SW];
    a = sqrtf((syy - sy * sy / sw) / (sxx - sx * sx / sw));
    b = (sy - a * sx) / sw;
}

// Pivoted LDL^T fallback (hostmath.h, Eigen's algorithm) for the rare case that the unpivoted solve meets a non-positive pivot.
// Out of line and fed from the sums in shared memory so that the fast path's matrices never have their address taken.
// `inline` for the linker only: tracking.cu and batches.cu both compile it.
__device__ __noinline__ inline void ldlt6SolvePivotedFromSums(const float* lsq, float lambda, float* incOut)
{
    static const unsigned char ij[21][2] = { {0,0},{0,1},{0,2},{0,3},{0,4},{0,5},{1,1},{1,2},{1,3},{1,4},{1,5},
                                            {2,2},{2,3},{2,4},{2,5},{3,3},{3,4},{3,5},{4,4},{4,5},{5,5} };
    float A[36], b[6];
    for (int k = 0; k < 21; k++) { const float v = lsq[k]; A[ij[k][0] * 6 + ij[k][1]] = v; A[ij[k][1] * 6 + ij[k][0]] = v; }
    for (int i = 0; i < 6; i++) b[i] = lsq[21 + i];
    const float damp = 1 + lambda;
    for (int i = 0; i < 6; i++) A[i * 6 + i] *= damp;
    lsd::ldlt6Solve(A, b, incOut);
}


// Solve the damped system `lsq` (RAW sums: LGS6::finish divides A and b by num_constraints, LGSX.h:319-325, which cancels
// in A^-1 b because the damping is multiplicative) and form exp(inc) * base with its rotation matrix (SE3Tracker.cpp:356-363).
__device__ __forceinline__ void solveCandidate(const float* lsq, float lambda, const lsd::SE3<float>& base, Cand& P, EvalPose& E, float affA, float affB)
{
    float A[36], b[6], inc[6];
    {
        int k = 0;
#pragma unroll
        for (int i = 0; i < 6; i++)
#pragma unroll
            for (int j = i; j < 6; j++) {
                const float v = lsq[k++];
                A[i * 6 + j] = v;
                A[j * 6 + i] = v;
            }
    }
#pragma unroll
    for (int i = 0; i < 6; i++) b[i] = lsq[21 + i];
    const float damp = 1 + lambda;
#pragma unroll
    for (int i = 0; i < 6; i++) A[i * 6 + i] *= damp;
    if (!ldltSolveFast<6>(A, b, inc)) {
        ldlt6SolvePivotedFromSums(lsq, lambda, P.inc);
#pragma unroll
        for (int i = 0; i < 6; i++) inc[i] = P.inc[i];
    }
    const lsd::SE3<float> c = se3ExpMulFast(inc, base);
    float dot = 0;
#pragma unroll
    for (int i = 0; i < 6; i++) { P.inc[i] = inc[i]; dot += inc[i] * inc[i]; }        // inc.dot(inc), :432
    P.incSq = dot;
    P.T = c;
    P.lambda = lambda;
    lsd::quatToMatrix(c.q, E.R);
    E.t[0] = c.t[0]; E.t[1] = c.t[1]; E.t[2] = c.t[2];
    E.a = affA; E.b = affB;
}

// std::pow(lambdaFailFac, incTry) of SE3Tracker.cpp:445 (float, int -> double pow): repeated multiplication in double,
// exact for the reference's factor 2 (and within an ulp of pow() for any other factor)
__device__ __forceinline__ double ipowd(double f, int n)
{
    double r = 1.0;
    for (int i = 0; i < n; i++) r *= f;
    return r;
}
// LM_lambda *= std::pow(lambdaFailFac, incTry), :445.  For the reference's factor 2 the product is an exact scaling by 2^n:
// one float multiply (FP64 issues at half the FP32 rate on H100 and this sits on the serial path of every pass).
__device__ __forceinline__ float lambdaAfterFail(float lambda, float failFac, int incTry)
{
    if (failFac == 2.0f && incTry >= 0 && incTry < 100 && lambda > 1e-30f && lambda < 1e8f)
        return lambda * __int_as_float((127 + incTry) << 23);
    return (float)((double)lambda * ipowd((double)failFac, incTry));
}

// Build the chain of the iteration that starts (or continues) now: lanes 0..kmax-1 of warp 0 solve, in parallel, for
// lambda_1 = lm.LM_lambda and its successors under rejection (lambda == 0 ? 0.2 : lambda * failFac^incTry, :443-446).
// The chain ends with the first candidate whose step is too small (its rejection ends the level, :432-441).
__device__ __forceinline__ void buildChain(const TrackParams& p, LMState& lm, LMShared& sh, int lane)
{
    const int lvl = lm.lvl;
    if (lane < p.kmax) {
        float lam = lm.LM_lambda;
        for (int u = 1; u <= lane; u++) {
            if (lam == 0) lam = 0.2f;
            else lam = lambdaAfterFail(lam, p.st.lambdaFailFac, lm.incTry + u);
        }
        solveCandidate(lm.lsq, lam, lm.refToFrame, sh.cand[lane], sh.pose[lane], lm.affine_a, lm.affine_b);
    }
    __syncwarp();
    if (lane == 0) {
        int K = 1;
        while (K < p.kmax && (sh.cand[K - 1].incSq > p.st.stepSizeMin[lvl])) K++;
        sh.nPose = K;
        lm.chainBase = lm.incTry;
        lm.phase = PH_TRY;
    }
}

__device__ __forceinline__ void lmNextLevel(const TrackParams& p, LMState& lm, LMShared& sh)
{
    lm.lvl--;
    if (lm.lvl < p.minLevel) { sh.action = ACT_LEVEL_DONE; return; }                // all levels done
    lm.phase = PH_INIT;
    setEvalPose(sh.pose[0], lm.refToFrame, lm.affine_a, lm.affine_b);
    sh.nPose = 1;
    sh.lvl = lm.lvl;
}

// Warp 0 after every pass: the decisions of SE3Tracker.cpp:324-446, replayed candidate by candidate in the reference's order.
// Lane 0 decides; all lanes of the warp take part in buildChain.
__device__ __forceinline__ void lmAdvance(const TrackParams& p, LMState& lm, LMShared& sh, int lane)
{
    int build = 0;                       // 1: start / continue an iteration (lane 0 decides, broadcast below)
    int copyLsq = 0;                     // 1: the sums of this pass become the accepted normal equations
    if (lane == 0) {
        const long long ta = clock64();
        const float* s = sh.sums;
        const int lvl = lm.lvl;
        const int K = sh.nPose;
        const float divTh = 0.01f * (p.W >> lvl) * (p.H >> lvl);     // MIN_GOODPERALL_PIXEL_ABSMIN is the float literal 0.01f (util/settings.h:170)
        sh.action = ACT_CONTINUE;
        lm.posesEvaluated += K;
        bool leave = false;
        // `accepted`: candidate 0 accepted with its normal equations at hand (init, re-evaluation or a first try)
        auto acceptActions = [&](bool init, float error) {
            if (!init) lm.refToFrame = lm.cand;
            if (p.useAffine) affineFromSums(s, lm.affine_a, lm.affine_b);               // :331-335 / :385-389
            const bool converged = !init && (error / lm.lastErr > p.st.convergenceEps[lvl]);   // :404
            if (!init) lm.last_residual = error;                                         // :414
            lm.lastErr = error;                                                          // :336 / :414
            copyLsq = 1;                                                                 // buffers now belong to this pose (all lanes copy below)
            if (init) { lm.LM_lambda = p.st.lambdaInitial[lvl]; lm.iteration = 0; }      // :341
            else {
                // :417-420 `if(LM_lambda <= 0.2)` compares the float with the DOUBLE 0.2 < 0.2f, i.e. LM_lambda < 0.2f
                if (lm.LM_lambda < 0.2f) lm.LM_lambda = 0;
                else lm.LM_lambda *= p.st.lambdaSuccessFac;
                if (!converged) lm.iteration++;
            }
            leave = converged || !(lm.iteration < p.st.maxItsPerLvl[lvl]);               // :343, :411
            if (!leave) { lm.nUpd[lvl]++; lm.incTry = 0; build = 1; }                    // calculateWarpUpdate(ls), :346
            lm.statsFrom = 0; lm.commitLast = 0;
        };
        if (lm.phase == PH_INIT || lm.phase == PH_REEVAL) {
            const float warped = s[CH_GOOD] + s[CH_BAD];
            if (lm.phase == PH_INIT && warped < divTh) {                                 // :324-329
                lm.diverged = 1; sh.action = ACT_DIVERGED; lm.statsFrom = 0; lm.commitLast = 0;
            } else {
                const float error = s[CH_SUMRESW] / warped;                              // calcWeightsAndResidual, :789
                if (lm.phase == PH_INIT) lm.nRes[lvl]++;                                 // a re-evaluated pose was counted when it was accepted
                acceptActions(lm.phase == PH_INIT, error);
            }
        } else {
            for (int k = 0; k < K; k++) {
                // sums of candidate k: main block (k == 0), last-candidate block (k == K-1) or the middle block
                const bool isLast = (k > 0 && k == K - 1);
                const float good = k == 0 ? s[CH_GOOD] : (isLast ? s[EV_NCH + XL_GOOD] : s[EV_NCH + XM_GOOD]);
                const float bad = k == 0 ? s[CH_BAD] : (isLast ? s[EV_NCH + XL_BAD] : s[EV_NCH + XM_BAD]);
                const float srw = k == 0 ? s[CH_SUMRESW] : (isLast ? s[EV_NCH + XL_SUMRESW] : s[EV_NCH + XM_SUMRESW]);
                const float warped = good + bad;
                lm.statsFrom = isLast ? 1 : 0;
                lm.commitLast = (isLast && lvl == SE3TRACKING_MIN_LEVEL) ? 1 : 0;     // only level 1 has a mask
                lm.cand = sh.cand[k].T;
#pragma unroll
                for (int i = 0; i < 6; i++) lm.inc[i] = sh.cand[k].inc[i];
                lm.LM_lambda = sh.cand[k].lambda;
                lm.incTry = lm.chainBase + k + 1;                                         // incTry++ after the solve, :361
                if (warped < divTh) {                                                    // :369-374
                    lm.diverged = 1; sh.action = ACT_DIVERGED;
                    break;
                }
                const float error = srw / warped;
                lm.nRes[lvl]++;
                if (error < lm.lastErr) {                                                // :381 accepted
                    if (k == 0) acceptActions(false, error);
                    else {
                        // a speculative candidate is the one the reference accepts: its normal equations and statistics were
                        // not accumulated -> evaluate it once more with all channels (same sums, bit for bit), then go on
                        lm.phase = PH_REEVAL;
                        setEvalPose(sh.pose[0], lm.cand, lm.affine_a, lm.affine_b);
                        sh.nPose = 1;
                    }
                    break;
                }
                // rejected, :424-447
                if (!(sh.cand[k].incSq > p.st.stepSizeMin[lvl])) { leave = true; break; }        // :432-441
                if (lm.LM_lambda == 0) lm.LM_lambda = 0.2f;                              // :443-446
                else lm.LM_lambda = lambdaAfterFail(lm.LM_lambda, p.st.lambdaFailFac, lm.incTry);
                if (k == K - 1) build = 1;                                               // chain used up: continue it
            }
        }
        if (leave) { lmNextLevel(p, lm, sh); build = 0; }
        if (sh.action != ACT_CONTINUE) build = 0;
        lm.dbg[0] += clock64() - ta;
    }
    build = __shfl_sync(0xffffffffu, build | (copyLsq << 1), 0);
    if (build & 2) {                     // 27 lanes instead of 27 dependent shared-memory round trips of lane 0
        if (lane < 27) lm.lsq[lane] = sh.sums[lane];
        __syncwarp();
    }
    build &= 1;
    if (build) {
        const long long tb = clock64();
        __syncwarp();
        buildChain(p, lm, sh, lane);
        if (lane == 0) lm.dbg[1] += clock64() - tb;
    }
}

// ---- batch layouts in the arena -------------------------------------------------------------------------------------------
// permaRef tracking (perma.cuh): one candidate descriptor / result per CTA
struct PermaItem {
    const float4* pc;                   // (x, y, z, colour) per point
    const float* var;                   // idepthVar per point
    int n;                              // permaRefNumPts
    float refToFrame[7];                // initial estimate, already cast to float (SE3Tracker.cpp:125,168)
};
struct PermaResult {
    float refToFrame[7];
    float pointUsage, goodCount, badCount, meanRes, lastResidual;
    float affine_a, affine_b;
    int diverged, nRes, nUpd;
};

// Sim3 tracking (sim3.cuh): one problem descriptor / result per cluster
#define S3_MAX_BATCH 1024

// reduction channels of one evaluation
enum {
    S3_A6 = 0,      // 21: upper triangle of sum v v^T wp            (LGS6::update, LGSX.h:390-396)
    S3_B6 = 21,     // 6:  sum v rp wp                               (LGS6::b = -this)
    S3_A4 = 27,     // 10: upper triangle of sum v4 v4^T wd          (LGS4::update, LGSX.h:163-169)
    S3_B4 = 37,     // 4:  sum v4 rd wd                              (LGS4::b = -this)
    S3_RESD = 41, S3_RESP = 42, S3_NUMD = 43, S3_NUMP = 44,          // Sim3ResidualStruct; numTermsP == buf_warped_size
    S3_USAGE = 45, S3_REFNUM = 46,
    S3_SXX = 47, S3_SYY = 48, S3_SX = 49, S3_SY = 50, S3_SW = 51,
    S3_NCH = 52
};
#define S3_NLGS 41                      // channels [0, 41) are the normal equations

struct Sim3Item {
    const float* kfIdepth[LSD_LEVELS];  // reference keyframe (the TrackingReference)
    const float* kfVar[LSD_LEVELS];
    const float4* kfGrad[LSD_LEVELS];   // (dx, dy, I, -): gradData and colour of makePointCloud in one texel
    const float4* frGrad[LSD_LEVELS];   // frame
    const float* frIdepth[LSD_LEVELS];
    const float* frVar[LSD_LEVELS];
    double refToFrame[7];               // initial referenceToFrame: scaled quaternion (x,y,z,w) + translation
};
struct Sim3Out {
    double refToFrame[7];
    float sums[S3_NCH];                 // the last evaluation
    float lgs[S3_NLGS];                 // normal-equation sums of the pose ls7 belongs to
    float resMean, resMeanD, resMeanP;  // finalResidual
    float pointUsage, affine_a, affine_b;
    int early;                          // 0: ok, 1: diverged (too few points), 2: increment out of range
    int nRes[LSD_LEVELS], nUpd[LSD_LEVELS];
    long long cyc[4];                   // thread-0 clock64 totals: pixel loop, CTA reduce, cluster exchange, serial LM step
};
