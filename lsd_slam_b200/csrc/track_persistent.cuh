// track_persistent.cuh -- SE3Tracker::trackFrame as ONE persistent cooperative kernel (mode 1).
//
// The whole coarse-to-fine Levenberg-Marquardt loop of Tracking/SE3Tracker.cpp:280-486 runs on the device:
// every CTA evaluates its share of the keyframe pixels with evalPoint() (track.cuh), the CTAs exchange their
// partial sums through L2 behind ONE grid-wide barrier per pass, and then EVERY CTA redundantly (and
// deterministically: same instructions on the same data) combines the partials in block order, takes the
// accept / reject / converge decisions of :381-446, solves the damped 6x6 systems (LDL^T) and applies
// exp(inc) * T.  No host round trip, no second barrier, no float atomics.  The host sees one launch and one
// 200-byte result per frame.
//
// CANDIDATE CHAINS.  Most of a pass is latency that no byte
// count touches (CTA reduction, ~5 dependent L2 round trips of barrier + combine, the serial LM step), and on the
// bench stream 10 of the 13 tries of a frame are REJECTED: after the first accepted step or two of a level the
// reference walks lambda = 0, 0.2, 0.8, 6.4, ... until the step is too small (:424-447).  All tries of one iteration
// share the normal equations, and lambda does not depend on the evaluations, so the whole chain is known the moment
// the iteration starts.  A pass therefore evaluates up to TP_KMAX poses: the try itself with all channels, and the
// next tries the reference would make if it rejects (error + counts; statistics for the chain's last pose).  The
// decisions are then replayed in the reference's order; whatever the reference would not have evaluated is
// discarded.  Results, call counters and the good-mask are exactly those of the one-pose-per-pass kernel (same
// per-point arithmetic, same reduction trees); only the number of passes drops (17 -> 11 on frame 1 of the stream).
//
// Why this shape: a 640x480 frame has <= 77k points on the finest tracked level, i.e. ~1 per resident
// thread; the reference's structure (3 loops per evaluation, one host decision between evaluations, 15-60
// evaluations per frame) is launch/latency bound by two orders of magnitude.  Grid = one CTA per SM (132 on an H100),
// co-residency guaranteed by the cooperative launch.
#pragma once
#include "internal.cuh"
#include "track.cuh"
#include <stdlib.h>
#include <atomic>

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

// Where a CTA sits in its launch.  The virtual grid has Gv = nRows * nRanks CTAs; the CTA walks row = b, b + Gs, ... < nRows and
// evaluates virtual CTA v = row * nRanks + rank into partial row `row`.  k_track_persistent: {blockIdx.x, gridDim.x, gridDim.x},
// one row per CTA (v = blockIdx.x * nRanks + rank); k_track_persistent_group: {blockIdx.x - s * Gs, Gs, Gv} with nRanks == 1.
struct SegGrid {
    int b;                           // physical CTA within the segment
    int Gs;                          // physical CTAs of the segment (the barrier counts these)
    int nRows;                       // partial rows the combine adds
};

// Grid-wide barrier.  Arrivals are counted on one word (monotonic: epoch e completes at base + e * gridDim arrivals, the
// counter is never reset): release-add, then polling of the counter itself; thread 0 carries the release / acquire for its
// CTA (cumulative over the __syncthreads on both sides).
__device__ __forceinline__ void gridBarrier(unsigned int* counter, unsigned int target)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned int v;
        asm volatile("atom.add.release.gpu.global.u32 %0, [%1], 1;" : "=r"(v) : "l"(counter) : "memory");
        if (v != target - 1u) {
            do {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
            } while ((int)(v - target) < 0);
        } else {
            asm volatile("fence.acq_rel.gpu;" ::: "memory");
        }
    }
    __syncthreads();
}

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

// Chunk (32 consecutive interior pixels) number `k` of CTA `b` on a grid of G CTAs.  A plain b + G*k would hand a CTA the
// same image columns in every slot (on the 320-wide level G = 132 chunks are 13.3 rows, so consecutive slots of a CTA lie almost
// exactly under one another): the semi-dense points cluster on textured structures, and the CTAs under them take longer than
// the mean, which every pass's barrier then waits for.  Rotating the assignment by a stride coprime to G per slot spreads a
// CTA's chunks over the columns.  Any bijection gives the same sums up to fp32 summation order (fixed for a given G).
__device__ __forceinline__ int tpChunkOf(int b, int k, int G)
{
    return k * G + (b + k * 37) % G;
}

// per-thread state carried in registers from one pass to the next
struct ThreadCarry {
    // the thread's first pixel of the current level, reconstructed once (see gridEvaluate)
    int pcLvl;
    bool pcIsPoint;
    float pcx, pcy, pcz, pcVar, pcColor;
};

// One pass: nPose candidate poses over this CTA's chunks of level `lvl`, CTA reduction, one row per CTA through L2 behind ONE
// grid barrier, then every CTA sums the rows in block order.  On return sh.sums holds the totals, bit-identical in every CTA.
// ---- one stream over several GPUs (BASELINE config 5): the per-pass sums cross NVLink inside the kernel ---------------------------
// After the local combine every CTA of this GPU holds this GPU's totals.  CTA 0 stores them, one 8-byte {value, tag} slot per
// channel, straight into every peer's exchange rows (peer-mapped memory: a posted NVLink write, no host, no NCCL call); every
// CTA then polls THE LOCAL copy of the peers' rows and adds the rows in rank order -- the same additions in the same order on
// every GPU, so all GPUs take the same LM decisions from identical bits.  Slots are double-buffered by pass parity: a row is
// overwritten two passes later, which needs this GPU's own next row, which CTA 0 sends only after every local CTA has passed the
// next local barrier, i.e. has consumed this one.
__device__ __forceinline__ void gridExchangeRanks(const TrackParams& p, LMShared& sh, int nch, unsigned int tag, unsigned int parity)
{
    const int t = threadIdx.x;
    if (t < nch) {
        const float mine = sh.sums[t];
        const size_t rowBase = (size_t)parity * TP_MAX_RANKS * 64;
        if (blockIdx.x == 0) {
            const unsigned long long w = ((unsigned long long)tag << 32) | __float_as_uint(mine);
            for (int d = 0; d < p.nRanks; d++) {
                if (d == p.rank) continue;
                unsigned long long* slot = reinterpret_cast<unsigned long long*>(p.peerSync[d] + TP_XCHG_OFFSET) + rowBase + p.rank * 64 + t;
                asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(slot), "l"(w) : "memory");
            }
        }
        float total = 0.f;
        for (int r = 0; r < p.nRanks; r++) {
            float v = mine;
            if (r != p.rank) {
                const unsigned long long* slot = reinterpret_cast<const unsigned long long*>(p.sync + TP_XCHG_OFFSET) + rowBase + r * 64 + t;
                unsigned long long w;
                do {
                    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(slot) : "memory");
                } while ((unsigned int)(w >> 32) != tag);
                v = __uint_as_float((unsigned int)w);
            }
            total = (r == 0) ? v : total + v;
        }
        sh.sums[t] = total;
    }
    __syncthreads();
}

// End of a sharded launch: when this kernel retires, (a) every level-1 flag this GPU wrote into its peers has landed and (b) every
// flag the peers wrote into this GPU has landed -- the mapping kernels that follow on each GPU's stream read the whole mask.
__device__ __forceinline__ void gridTailRanks(const TrackParams& p)
{
    __threadfence_system();                                   // this thread's peer stores are performed system-wide
    gridBarrier(p.sync + TP_TAIL_OFFSET, p.tailBase + gridDim.x);
    if (blockIdx.x != 0) return;
    const int d = threadIdx.x;
    if (d < p.nRanks && d != p.rank) {
        const unsigned long long tag = ((unsigned long long)p.launchSeq << 32) | 0xd0d0d0d0ull;
        unsigned long long* theirs = reinterpret_cast<unsigned long long*>(p.peerSync[d] + TP_DONE_OFFSET) + p.rank;
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(theirs), "l"(tag) : "memory");
        const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(p.sync + TP_DONE_OFFSET) + d;
        unsigned long long w;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(mine) : "memory");
        } while (w != tag);
    }
    __syncthreads();
}

__device__ __forceinline__ void gridEvaluate(const TrackParams& p, const SegGrid& sg, int lvl, LMShared& sh, float (*sm)[EV_NCHX],
                                             float (*comb)[TP_ROW], unsigned int& epoch, long long* cyc, ThreadCarry& tc)
{
    long long t0 = clock64(), t1;
    const TrackLevelParams& L = p.lvl[lvl];
    const int K = sh.nPose;
    const EvalPose P = sh.pose[0];
    const int w = L.w, h = L.h, iw = L.iw, nInt = L.nInt;
    const float4* fg = L.frameGrad;
    uint8_t* mask = (lvl == SE3TRACKING_MIN_LEVEL) ? p.goodMask : nullptr;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // chunks of virtual CTA v: tpChunkOf(v, k, Gv), k = 0 .. nSlots-1 where it exists; warp `warp` takes k = warp, warp + 16, ...
    // The CTA runs the virtual CTAs of its rows in turn (SegGrid); sharded over nRanks GPUs, the CTAs of all ranks form one
    // virtual grid.
    const int Gv = sg.nRows * p.nRanks;
    const int nSlots = (L.nChunks + Gv - 1) / Gv;
    const int nch = K > 1 ? EV_NCHX : EV_NCH;
    const unsigned int parity = epoch & 1u;
    float* part = p.partials + (size_t)parity * TP_ROW * sg.nRows;
    int row = sg.b;
    do {
        const int vb = row * p.nRanks + p.rank;
        PointAcc acc;
        float ext[EV_NX];
#pragma unroll
        for (int c = 0; c < EV_NCH; c++) acc.v[c] = 0.f;
#pragma unroll
        for (int c = 0; c < EV_NX; c++) ext[c] = 0.f;
        for (int k = warp; k < nSlots; k += TP_WARPS) {
            const int chunk = tpChunkOf(vb, k, Gv);
            if (chunk >= L.nChunks) continue;                              // warp-uniform
            const int j = (chunk << 5) + lane;                             // interior pixel number
            const bool firstChunk = k == warp && row == sg.b;              // the point cache holds the first virtual CTA's pixel
            bool isPoint = false;
            float px = 0.f, py = 0.f, pz = 0.f, var = 0.f, color = 0.f;
            int i = 0;
            if (j < nInt) {
                const int yy = j / iw;
                i = (j - yy * iw + 1) + (yy + 1) * w;                      // x = 1 + j % iw, y = 1 + j / iw
            }
            if (firstChunk && tc.pcLvl == lvl) {
                // the thread's first pixel of a level never changes between the passes of that level: keep the
                // reconstructed point in registers instead of re-reading the keyframe planes (an L2 round trip at the head
                // of every pass's dependency chain)
                isPoint = tc.pcIsPoint; px = tc.pcx; py = tc.pcy; pz = tc.pcz; var = tc.pcVar; color = tc.pcColor;
            } else {
                if (j < nInt) {
                    const float idepth = __ldg(L.kfIdepth + i);
                    var = __ldg(L.kfVar + i);
                    if (!(var <= 0 || idepth == 0)) {                      // TrackingReference.cpp:133
                        const int yy = j / iw, x = j - yy * iw + 1, y = yy + 1;
                        const float sc = 1.0f / idepth;
                        px = sc * (L.fxi * x + L.cxi); py = sc * (L.fyi * y + L.cyi); pz = sc * 1;
                        color = __ldg(L.kfColor + i);
                        isPoint = true;
                    }
                }
                if (firstChunk) {
                    tc.pcLvl = lvl; tc.pcIsPoint = isPoint;
                    tc.pcx = px; tc.pcy = py; tc.pcz = pz; tc.pcVar = var; tc.pcColor = color;
                }
            }
            if (isPoint) {
                auto tap = [fg, w](float u, float v, float& o0, float& o1, float& o2) { interp43(fg, u, v, w, o0, o1, o2); };
                const int good = evalPoint(px, py, pz, color, var, P, p.C, L.fx, L.fy, L.cx, L.cy, w, h, tap, acc);
                if (K > 1) {                                               // block-uniform
                    if (K > 2) evalPointLight<false>(px, py, pz, color, var, sh.pose[1], p.C, L.fx, L.fy, L.cx, L.cy, w, h, tap, ext);
                    const int goodL = evalPointLight<true>(px, py, pz, color, var, sh.pose[K - 1], p.C, L.fx, L.fy, L.cx, L.cy, w, h, tap, ext);
                    if (mask) p.lastMask[i] = (uint8_t)goodL;
                }
                if (mask) {
                    mask[i] = (uint8_t)good;
                    if (p.nRanks > 1)                                      // the other ranks own other chunks: give them this one's flag
                        for (int d = 0; d < p.nRanks; d++) if (d != p.rank) p.peerMask[d][i] = (uint8_t)good;
                }
            }
        }
        __syncthreads();
        t1 = clock64();
        if (K > 1) warpReduceExt(ext, lane, sm[warp]);                    // first: its 16 registers are free for the 40 channels
        warpReduceAcc(acc, lane, sm[warp]);
        __syncthreads();
        float ctaSum = 0.f;
        if (threadIdx.x < nch) {
#pragma unroll
            for (int wi = 0; wi < TP_WARPS; wi++) ctaSum += sm[wi][threadIdx.x];
        }
        // ---- exchange: ONE 256-byte row per CTA ([parity][cta][64 floats], written through to L2 as one coalesced store),
        // ONE grid barrier, then every CTA combines all rows in a fixed order.  (Round 1 laid the buffer out [channel][cta]:
        // 40 four-byte writes per CTA into lines shared with 31 other CTAs -- 5 920 partial-sector writes per pass behind the
        // release of the barrier, and the combine's loads then waited ~5 000 cycles on those lines: 25 % of the kernel, ncu.)
        // A CTA with several rows writes each of them; the next one reuses sm only after the __syncthreads that ends its chunk loop.
        if (threadIdx.x < nch) __stcg(part + (size_t)row * TP_ROW + threadIdx.x, ctaSum);
        row += sg.Gs;
    } while (row < sg.nRows);
    epoch++;
    long long t2 = clock64();
    gridBarrier(p.sync, p.barrierBase + epoch * (unsigned int)sg.Gs);
    long long t3 = clock64();
    // warp wi adds rows wi, wi+16, ... (<= 10): the lower half-warp takes the even ones of those, the upper half the odd ones, each
    // lane one float4 (4 channels) of a 256-byte row -- 5 vector loads per thread, all in flight before the first add.  fp32 adds
    // in a fixed order (rows ascending per half-warp, then upper half onto lower, then the 16 warps in order): every CTA executes
    // the same additions in the same order on the same data, so the totals are bit-identical everywhere, and the sums stay in
    // the precision the per-point accumulators and the reference's own (sequential fp32) sums have.
    {
        const int nb = sg.nRows;
        const int half = lane >> 4, q = lane & 15;
        constexpr int NR = (TP_MAXGRID / TP_WARPS + 1) / 2;
        float4 v[NR];
#pragma unroll
        for (int r = 0; r < NR; r++) {
            const int row = warp + (2 * r + half) * TP_WARPS;
            v[r] = (row < nb) ? __ldcg(reinterpret_cast<const float4*>(part + (size_t)row * TP_ROW) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float4 a = v[0];
#pragma unroll
        for (int r = 1; r < NR; r++) { a.x += v[r].x; a.y += v[r].y; a.z += v[r].z; a.w += v[r].w; }
        a.x += __shfl_down_sync(0xffffffffu, a.x, 16);
        a.y += __shfl_down_sync(0xffffffffu, a.y, 16);
        a.z += __shfl_down_sync(0xffffffffu, a.z, 16);
        a.w += __shfl_down_sync(0xffffffffu, a.w, 16);
        if (half == 0) reinterpret_cast<float4*>(&comb[warp][0])[q] = a;
    }
    __syncthreads();
    if (threadIdx.x < nch) {
        float t = comb[0][threadIdx.x];
#pragma unroll
        for (int wi = 1; wi < TP_WARPS; wi++) t += comb[wi][threadIdx.x];
        sh.sums[threadIdx.x] = t;
    }
    __syncthreads();
    if (p.nRanks > 1) gridExchangeRanks(p, sh, nch, (p.launchSeq << 16) | (epoch & 0xffffu), epoch & 1u);
    long long t4 = clock64();
    cyc[0] += t1 - t0; cyc[1] += t2 - t1; cyc[2] += t3 - t2; cyc[3] += t4 - t3;
}

// Fully unrolled, register-resident LDL^T (no pivoting) for the damped 6x6 normal equations.  Returns false if
// a pivot is not strictly positive (then the caller falls back to the pivoted routine, hostmath.h).
__device__ __forceinline__ bool ldlt6SolveFast(const float* A, const float* b, float* x)
{
    float L[6][6], D[6];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 6; j++) {
        float d = A[j * 6 + j];
#pragma unroll
        for (int k = 0; k < j; k++) d -= L[j][k] * L[j][k] * D[k];
        D[j] = d;
        ok = ok && (d > 0.f);
        const float inv = 1.0f / d;
#pragma unroll
        for (int i = j + 1; i < 6; i++) {
            float v = A[i * 6 + j];
#pragma unroll
            for (int k = 0; k < j; k++) v -= L[i][k] * L[j][k] * D[k];
            L[i][j] = v * inv;
        }
    }
    float y[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        float s = b[i];
#pragma unroll
        for (int k = 0; k < i; k++) s -= L[i][k] * y[k];
        y[i] = s;
    }
#pragma unroll
    for (int i = 0; i < 6; i++) y[i] = y[i] / D[i];
#pragma unroll
    for (int i = 5; i >= 0; i--) {
        float s = y[i];
#pragma unroll
        for (int k = i + 1; k < 6; k++) s -= L[k][i] * x[k];
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
__device__ __noinline__ void ldlt6SolvePivotedFromSums(const float* lsq, float lambda, float* incOut)
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
    if (!ldlt6SolveFast(A, b, inc)) {
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

// The tracker of one stream on the CTAs `sg` describes: the whole grid (k_track_persistent) or one segment of a group launch
// (k_track_persistent_group).  Both run the same passes, decisions and combine.
__device__ __forceinline__ void trackStream(const TrackParams& p, TrackState* __restrict__ out, const SegGrid& sg)
{
    __shared__ alignas(LMShared) unsigned char shStorage[sizeof(LMShared)];   // raw storage: Cand holds a type with a constructor
    LMShared& sh = *reinterpret_cast<LMShared*>(shStorage);
    __shared__ alignas(LMState) unsigned char lmStorage[sizeof(LMState)];     // every field is written before use; no constructor in shared memory
    LMState& lm = *reinterpret_cast<LMState*>(lmStorage);
    __shared__ float sm[TP_WARPS][EV_NCHX];
    __shared__ __align__(16) float comb[TP_WARPS][TP_ROW];         // per-warp partial sums of the combine
    static_assert(EV_NCH == 40 && EV_NX == 16, "warpReduceAcc / warpReduceExt are written for 32 + 8 (+ 16) channels");
    unsigned int epoch = 0;
    long long cyc[6] = { 0, 0, 0, 0, 0, 0 };
    const long long tStart = clock64();
    ThreadCarry tc;
    tc.pcLvl = -1; tc.pcIsPoint = false;
    tc.pcx = tc.pcy = tc.pcz = tc.pcVar = tc.pcColor = 0.f;

    // fresh refPixelWasGood mask: all true (Frame.h:433); ordered before the level-1 passes by the barriers
    if (p.maskFresh) {
        uint32_t* m32 = reinterpret_cast<uint32_t*>(p.goodMask);
        for (int i = sg.b * TP_THREADS + threadIdx.x; i < p.maskBytes / 4; i += sg.Gs * TP_THREADS) m32[i] = 0x01010101u;
    }

    if (threadIdx.x == 0) {
        for (int i = 0; i < 4; i++) lm.refToFrame.q[i] = p.initRefToFrame[i];
        for (int i = 0; i < 3; i++) lm.refToFrame.t[i] = p.initRefToFrame[4 + i];
        for (int l = 0; l < LSD_LEVELS; l++) { lm.nRes[l] = 0; lm.nUpd[l] = 0; lm.nEval[l] = 0; lm.nPts[l] = 0.f; }
        lm.affine_a = 1.f; lm.affine_b = 0.f; lm.lastErr = 0.f; lm.last_residual = 0.f; lm.LM_lambda = 0.f;
        lm.diverged = 0; lm.incTry = 0; lm.iteration = 0; lm.dbg[0] = lm.dbg[1] = lm.dbg[2] = lm.dbg[3] = 0;
        lm.chainBase = 0; lm.statsFrom = 0; lm.commitLast = 0; lm.posesEvaluated = 0;
        lm.lvl = SE3TRACKING_MAX_LEVEL - 1; lm.phase = PH_INIT;
        sh.lvl = lm.lvl; sh.action = ACT_CONTINUE; sh.nPose = 1;
        setEvalPose(sh.pose[0], lm.refToFrame, lm.affine_a, lm.affine_b);
    }
    __syncthreads();

    while (true) {
        const int lvl = sh.lvl;
        gridEvaluate(p, sg, lvl, sh, sm, comb, epoch, cyc, tc);
        if (threadIdx.x < 32) {
            if (threadIdx.x == 0) { lm.nEval[lvl]++; lm.nPts[lvl] = sh.sums[CH_REFNUM]; }
            lmAdvance(p, lm, sh, threadIdx.x);
        }
        __syncthreads();
        if (sh.action != ACT_CONTINUE) break;
    }

    // The mask holds the flags of candidate 0 of the last level-1 pass; if the last pose the reference evaluates was the chain's
    // last candidate instead, its flags (p.lastMask) replace them now.  Same threads, same pixels: no synchronisation.
    if (lm.commitLast && p.minLevel == SE3TRACKING_MIN_LEVEL) {
        // this thread wrote p.lastMask in the last pass for every point it evaluated; the points are found again from the keyframe
        // planes (the test of gridEvaluate), row by row of the CTA as gridEvaluate walks them
        const TrackLevelParams& L = p.lvl[SE3TRACKING_MIN_LEVEL];
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        const int Gv = sg.nRows * p.nRanks;
        const int nSlots = (L.nChunks + Gv - 1) / Gv;
        for (int row = sg.b; row < sg.nRows; row += sg.Gs)
            for (int k = warp; k < nSlots; k += TP_WARPS) {
                const int j = (tpChunkOf(row * p.nRanks + p.rank, k, Gv) << 5) + lane;
                if (j >= L.nInt) continue;
                const int yy = j / L.iw;
                const int i = (j - yy * L.iw + 1) + (yy + 1) * L.w;
                const float idepth = L.kfIdepth[i], var = L.kfVar[i];
                if (var <= 0 || idepth == 0) continue;
                const uint8_t g = p.lastMask[i];
                p.goodMask[i] = g;
                if (p.nRanks > 1)
                    for (int d = 0; d < p.nRanks; d++) if (d != p.rank) p.peerMask[d][i] = g;
            }
    }
    if (p.nRanks > 1) gridTailRanks(p);

    // the per-CTA cycle table (LSDGPU_TRACK_DEBUG) is written by single-stream launches only (fillTrackParams leaves debug 0)
    if (p.debug && threadIdx.x == 0 && sg.b < TP_MAXGRID - 1) {
        long long tot = clock64() - tStart;
        for (int i = 0; i < 4; i++) out->cycBlk[sg.b][i] = cyc[i];
        out->cycBlk[sg.b][5] = tot;
        out->cycBlk[sg.b][4] = tot - cyc[0] - cyc[1] - cyc[2] - cyc[3];
    }
    if (sg.b == 0 && threadIdx.x == 0) {
        // statistics of the LAST EVALUATED pose (SURVEY App. A-1): main block, or the extension block's last candidate
        float fin[EV_NCH];
        for (int c = 0; c < EV_NCH; c++) fin[c] = sh.sums[c];
        if (lm.statsFrom == 1) {
            const float* x = sh.sums + EV_NCH;
            fin[CH_SUMRESW] = x[XL_SUMRESW]; fin[CH_SUMRESU] = x[XL_SUMRESU]; fin[CH_SIGNED] = x[XL_SIGNED];
            fin[CH_GOOD] = x[XL_GOOD]; fin[CH_BAD] = x[XL_BAD]; fin[CH_USAGE] = x[XL_USAGE];
            fin[CH_SXX] = x[XL_SXX]; fin[CH_SYY] = x[XL_SYY]; fin[CH_SX] = x[XL_SX]; fin[CH_SY] = x[XL_SY]; fin[CH_SW] = x[XL_SW];
        }
        lsdgpu_eval_result ev;
        evalFinish(fin, &ev);
        for (int i = 0; i < 4; i++) out->refToFrame[i] = lm.refToFrame.q[i];
        for (int i = 0; i < 3; i++) out->refToFrame[4 + i] = lm.refToFrame.t[i];
        out->pointUsage = ev.pointUsage; out->goodCount = ev.goodCount; out->badCount = ev.badCount;
        out->meanRes = ev.meanRes; out->lastResidual = lm.last_residual;
        out->affine_a = lm.affine_a; out->affine_b = lm.affine_b;
        out->diverged = lm.diverged;
        for (int l = 0; l < LSD_LEVELS; l++) {
            out->numCalcResidualCalls[l] = lm.nRes[l]; out->numCalcWarpUpdateCalls[l] = lm.nUpd[l]; out->evalsAtLevel[l] = lm.nEval[l];
            out->pointsAtLevel[l] = lm.nPts[l];
        }
        out->posesEvaluated = lm.posesEvaluated;
        out->totalEvals = (int)epoch;
        cyc[5] = clock64() - tStart;
        cyc[4] = cyc[5] - cyc[0] - cyc[1] - cyc[2] - cyc[3];
        for (int i = 0; i < 6; i++) out->cyc[i] = cyc[i];
        if (p.debug) for (int i = 0; i < 4; i++) out->cycBlk[TP_MAXGRID - 1][i] = lm.dbg[i];
        __threadfence_system();
        out->doneSeq = p.launchSeq;
    }
}

__global__ void __launch_bounds__(TP_THREADS, 1) k_track_persistent(const __grid_constant__ TrackParams p, TrackState* __restrict__ out)
{
    trackStream(p, out, SegGrid{ (int)blockIdx.x, (int)gridDim.x, (int)gridDim.x });
}

// n streams in one cooperative launch of n * Gs CTAs: CTAs [s * Gs, (s + 1) * Gs) track segs[s] on a virtual grid of Gv CTAs
__global__ void __launch_bounds__(TP_THREADS, 1) k_track_persistent_group(const TrackGroupSeg* __restrict__ segs, int Gs, int Gv)
{
    const int s = (int)blockIdx.x / Gs;
    const TrackGroupSeg& g = segs[s];
    trackStream(g.p, g.out, SegGrid{ (int)blockIdx.x - s * Gs, Gs, Gv });
}

static cudaError_t trackPersistentSetup(lsdgpu_ctx* ctx)
{
    int coop = 0;
    cudaError_t e = cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, ctx->device);
    if (e != cudaSuccess) return e;
    if (!coop) return cudaErrorNotSupported;
    ctx->optTrackDebug = getenv("LSDGPU_TRACK_DEBUG") != nullptr;              // read once, not per frame
    ctx->trackGrid = ctx->smCount < TP_MAXGRID ? ctx->smCount : TP_MAXGRID;      // one CTA per SM, co-resident (cooperative launch)
    if (ctx->optTrackDebug) fprintf(stderr, "[track] grid %d, candidate poses per pass <= %d\n", ctx->trackGrid, TP_KMAX);
    return cudaSuccess;
}

// device time of the last profiled tracking launch (CUDA events on the context's stream), accumulated lazily
static void flushTrackProfile(lsdgpu_ctx* ctx)
{
    if (!ctx->trackProfilePending) return;
    float ms = 0;
    cudaEventSynchronize(ctx->kEnd);
    if (cudaEventElapsedTime(&ms, ctx->kBegin, ctx->kEnd) == cudaSuccess) { ctx->trackKernelMs += ms; ctx->trackKernelLaunches++; }
    ctx->trackProfilePending = false;
}

// one cooperative launch of a tracking kernel (every CTA co-resident: the grid barrier relies on it)
static cudaError_t launchCooperative(const void* kernel, int grid, cudaStream_t stream, void** args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(TP_THREADS); cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelExC(&cfg, kernel, args);
}

// the parameters of one frame's tracking on this context (single-GPU part; trackPersistent adds the peers of a sharded stream)
static void fillTrackParams(lsdgpu_ctx* ctx, FrameSlot* kf, FrameSlot* fr, const double init_qt[7], const lsdgpu_track_settings* st,
                            TrackParams& P)
{
    memset(&P, 0, sizeof(P));
    for (int l = SE3TRACKING_MIN_LEVEL; l < SE3TRACKING_MAX_LEVEL; l++) {
        const LevelCam& c = ctx->cam[l];
        TrackLevelParams& L = P.lvl[l];
        L.kfIdepth = kf->idepth[l]; L.kfVar = kf->idepthVar[l]; L.kfColor = kf->image[l]; L.frameGrad = fr->grad[l];
        L.w = c.w; L.h = c.h; L.fx = c.fx; L.fy = c.fy; L.cx = c.cx; L.cy = c.cy;
        L.fxi = c.fxi; L.fyi = c.fyi; L.cxi = c.cxi; L.cyi = c.cyi;
        // no interior on a level 1 or 2 pixels wide or high (1x1 at 16x16): (w-2)*(h-2) would count (-1)*(-1) = 1 point
        L.iw = c.w - 2; L.nInt = std::max(c.w - 2, 0) * std::max(c.h - 2, 0); L.nChunks = (L.nInt + 31) / 32;
    }
    P.lastMask = ctx->dLastMask;
    P.minLevel = SE3TRACKING_MIN_LEVEL;
    P.goodMask = fr->goodMask;
    P.maskFresh = fr->hasGoodMask ? 0 : 1;
    P.maskBytes = (ctx->w * ctx->h) / 4;
    P.W = ctx->w; P.H = ctx->h;
    lsd::SE3<double> init;
    for (int i = 0; i < 4; i++) init.q[i] = init_qt[i];
    for (int i = 0; i < 3; i++) init.t[i] = init_qt[4 + i];
    lsd::SE3<float> r2f = lsd::se3Cast<float>(lsd::se3Inverse(init));             // SE3Tracker.cpp:306
    for (int i = 0; i < 4; i++) P.initRefToFrame[i] = r2f.q[i];
    for (int i = 0; i < 3; i++) P.initRefToFrame[4 + i] = r2f.t[i];
    P.st = *st;
    P.C.cameraPixelNoise2 = ctx->g.cameraPixelNoise2; P.C.var_weight = st->var_weight; P.C.huber_half = st->huber_d / 2;
    P.useAffine = ctx->g.useAffineLightningEstimation;
    P.partials = ctx->evPartials;
    P.sync = ctx->trkSync;
    P.barrierBase = ctx->trkBase;
    P.kmax = TP_KMAX;
    P.nRanks = 1; P.rank = 0;
}

// Wait for the result block of launch `ctx->trackSeq`, spinning on its sequence word (a few hundred ns of latency) instead of a stream
// synchronisation; `launchStream` is the stream the kernel was launched on.
static int waitTrackState(lsdgpu_ctx* ctx, cudaStream_t launchStream)
{
    TrackState* hOut = (TrackState*)ctx->hTrackState;
    bool done = false;
    for (long long spin = 0; spin < 200000000LL; spin++) {
        if (hOut->doneSeq == ctx->trackSeq) { done = true; break; }
        if ((spin & 0xffff) == 0xffff && cudaStreamQuery(launchStream) != cudaErrorNotReady) { done = hOut->doneSeq == ctx->trackSeq; break; }
    }
    if (!done) LSD_CHECK(ctx, cudaStreamSynchronize(launchStream));
    // the other fields of the mapped result block are read with plain loads afterwards: keep them behind the doneSeq read.  Block 0
    // publishes doneSeq while other CTAs may still be exiting, so only STREAM-ORDERED consumers may assume the kernel has retired.
    std::atomic_thread_fence(std::memory_order_acquire);
    return 0;
}

// SURVEY 8d, fused single-pass kernel: B_fused(l) = 20 B per valid point + 16 B per texel of the frame's gradient
// level (+5 B per point on L1: mask byte + index) + 160 B of partial sums, per evaluation OF THE REFERENCE
// (numCalcResidualCalls; speculative candidates the reference would not evaluate are not counted).  The kernel reads the
// three keyframe planes densely (12 B per pixel); the ALGORITHMIC figure charges only the valid points, as the survey defines it.
static double trackAlgorithmicBytes(const lsdgpu_ctx* ctx, const TrackState* hOut)
{
    double bytes = 0;
    for (int l = SE3TRACKING_MIN_LEVEL; l < SE3TRACKING_MAX_LEVEL; l++) {
        const double np_ = (double)hOut->pointsAtLevel[l];   // numData[level]: valid points of the level (CH_REFNUM)
        bytes += (double)hOut->numCalcResidualCalls[l] * (20.0 * np_ + 16.0 * (double)ctx->cam[l].w * ctx->cam[l].h + (l == 1 ? 5.0 * np_ : 0.0) + EV_NCH * 4.0);
    }
    return bytes;
}

// the result block -> SE3Tracker's public fields (SE3Tracker.cpp:453-485)
static void translateTrackState(const lsdgpu_ctx* ctx, const TrackState* hOut, lsdgpu_track_result* out)
{
    out->pointUsage = hOut->pointUsage; out->lastGoodCount = hOut->goodCount; out->lastBadCount = hOut->badCount;
    out->lastMeanRes = hOut->meanRes;
    out->affineEstimation_a = hOut->affine_a; out->affineEstimation_b = hOut->affine_b;
    for (int l = 0; l < LSD_LEVELS; l++) {
        out->numCalcResidualCalls[l] = hOut->numCalcResidualCalls[l];
        out->numCalcWarpUpdateCalls[l] = hOut->numCalcWarpUpdateCalls[l];
    }
    if (hOut->diverged) {
        out->frameToRef_qt[3] = 1;
        out->diverged = 1; out->trackingWasGood = 0;
        return;
    }
    const int W = ctx->w, H = ctx->h;
    out->lastResidual = hOut->lastResidual;
    out->trackingWasGood = hOut->goodCount / ((W >> SE3TRACKING_MIN_LEVEL) * (H >> SE3TRACKING_MIN_LEVEL)) > 0.04f
                           && hOut->goodCount / (hOut->goodCount + hOut->badCount) > 0.5f;
    out->initialTrackedResidual = out->lastResidual / out->pointUsage;
    lsd::SE3<float> T;
    for (int i = 0; i < 4; i++) T.q[i] = hOut->refToFrame[i];
    for (int i = 0; i < 3; i++) T.t[i] = hOut->refToFrame[4 + i];
    lsd::SE3<double> f2r = lsd::se3Cast<double>(lsd::se3Inverse(T));
    for (int i = 0; i < 4; i++) out->frameToRef_qt[i] = f2r.q[i];
    for (int i = 0; i < 3; i++) out->frameToRef_qt[4 + i] = f2r.t[i];
}

// a stream's completed launch: its barrier counted `barrierCtas` arrivals per pass (the counter is never reset), and its result
// block becomes `out`
static void trackLaunchDone(lsdgpu_ctx* ctx, unsigned int barrierCtas, lsdgpu_track_result* out)
{
    const TrackState* hOut = (const TrackState*)ctx->hTrackState;
    ctx->trkBase += (unsigned int)hOut->totalEvals * barrierCtas;
    translateTrackState(ctx, hOut, out);
}

// track one frame: launch the kernel on the context's stream, wait for its result block and translate it (SE3Tracker.cpp:453-485)
static int trackPersistent(lsdgpu_ctx* ctx, FrameSlot* kf, FrameSlot* fr, const double init_qt[7],
                           const lsdgpu_track_settings* st, lsdgpu_track_result* out)
{
    flushTrackProfile(ctx);
    TrackParams P;
    fillTrackParams(ctx, kf, fr, init_qt, st, P);
    P.nRanks = ctx->nRanks; P.rank = ctx->rank;
    P.tailBase = ctx->trkTailBase;
    for (int d = 0; d < ctx->nRanks; d++) {
        char* base = d == ctx->rank ? ctx->arena : ctx->peerBase[d];
        P.peerSync[d] = reinterpret_cast<unsigned int*>(base + ((char*)ctx->trkSync - ctx->arena));
        P.peerMask[d] = reinterpret_cast<uint8_t*>(base + ((char*)fr->goodMask - ctx->arena));
    }
    if (ctx->nRanks > 1) ctx->trkTailBase += (unsigned int)ctx->trackGrid;
    TrackState* dOut = (TrackState*)ctx->dTrackStateMapped;

    void* args[] = { (void*)&P, (void*)&dOut };
    P.debug = ctx->optTrackDebug ? 1 : 0;
    P.launchSeq = ++ctx->trackSeq;
    if (ctx->profileTrackKernel) cudaEventRecord(ctx->kBegin, ctx->stream);
    LSD_CHECK(ctx, launchCooperative((const void*)k_track_persistent, ctx->trackGrid, ctx->stream, args));    // one CTA per SM
    ctx->launches++;
    if (ctx->profileTrackKernel) cudaEventRecord(ctx->kEnd, ctx->stream);
    fr->hasGoodMask = true;

    memset(out, 0, sizeof(*out));
    TrackState* hOut = (TrackState*)ctx->hTrackState;
    // The result block lives in mapped pinned memory and its last word is a sequence number: spin on it (a few
    // hundred ns of latency) instead of a stream synchronisation.  Later launches are stream-ordered anyway.
    if (ctx->optTrackDebug) {
        LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
        std::atomic_thread_fence(std::memory_order_acquire);
    } else {
        const int r = waitTrackState(ctx, ctx->stream);
        if (r) return r;
    }
    trackLaunchDone(ctx, (unsigned int)ctx->trackGrid, out);

    if (ctx->profileTrackKernel) {           // the event pair is read lazily (flushTrackProfile): no extra sync on the path
        ctx->trackKernelBytes += trackAlgorithmicBytes(ctx, hOut);
        ctx->trackProfilePending = true;
    }

    if (ctx->optTrackDebug) {
        fprintf(stderr, "[track] passes=%d (L4..L1: %d %d %d %d) poses=%d reference evaluations=%d cycles: points=%lld ctaReduce=%lld barrier=%lld combine=%lld serialLM=%lld total=%lld\n",
                hOut->totalEvals, hOut->evalsAtLevel[4], hOut->evalsAtLevel[3], hOut->evalsAtLevel[2], hOut->evalsAtLevel[1], hOut->posesEvaluated,
                hOut->numCalcResidualCalls[4] + hOut->numCalcResidualCalls[3] + hOut->numCalcResidualCalls[2] + hOut->numCalcResidualCalls[1],
                hOut->cyc[0], hOut->cyc[1], hOut->cyc[2], hOut->cyc[3], hOut->cyc[4], hOut->cyc[5]);
        fprintf(stderr, "   warp 0: decisions=%lld chain building=%lld\n", hOut->cycBlk[TP_MAXGRID - 1][0], hOut->cycBlk[TP_MAXGRID - 1][1]);
        const char* nm[6] = { "points", "ctaReduce", "barrier", "combine", "serial", "total" };
        const int gAll = ctx->trackGrid;
        for (int k = 0; k < 6; k++) {
            long long mn = 1LL << 60, mx = 0, sum = 0; int imx = 0, imn = 0;
            for (int b = 0; b < gAll && b < TP_MAXGRID - 1; b++) {
                long long v = hOut->cycBlk[b][k];
                if (v < mn) { mn = v; imn = b; }
                if (v > mx) { mx = v; imx = b; }
                sum += v;
            }
            fprintf(stderr, "   %-9s min=%lld (cta %d) max=%lld (cta %d) mean=%lld\n", nm[k], mn, imn, mx, imx, sum / gAll);
        }
        if (getenv("LSDGPU_TRACK_DEBUG_CTAS")) {
            for (int k = 0; k < 3; k++) {
                fprintf(stderr, "   %s per cta:", nm[k]);
                for (int b = 0; b < gAll && b < TP_MAXGRID - 1; b++) fprintf(stderr, " %lld", hOut->cycBlk[b][k] / 100);
                fprintf(stderr, "\n");
            }
        }
    }
    return 0;
}

// Track the frames of n contexts on one device in ONE cooperative launch of k_track_persistent_group on ctxs[0]'s stream.  The
// caller has enqueued every frame's construction on its own context's stream: the launching stream waits for all of them, and every
// other stream waits for the launch, so that each context's later work stays ordered after its tracking.
// On an error, *failed is the index of the context whose message is set.
static int trackPersistentGroup(int n, lsdgpu_ctx* const* ctxs, FrameSlot* const* kfs, FrameSlot* const* frs, const double* const* initQts,
                                const lsdgpu_track_settings* const* sts, lsdgpu_track_result* outs, int* failed)
{
    lsdgpu_ctx* c0 = ctxs[0];
    int Gs = c0->trackGrid / n, Gv = c0->trackGrid;
    TrackGroupSeg* h = (TrackGroupSeg*)c0->hGroupSegs;
    for (int i = 0; i < n; i++) {
        lsdgpu_ctx* ctx = ctxs[i];
        *failed = i;
        flushTrackProfile(ctx);
        fillTrackParams(ctx, kfs[i], frs[i], initQts[i], sts[i], h[i].p);
        h[i].p.launchSeq = ++ctx->trackSeq;
        h[i].out = (TrackState*)ctx->dTrackStateMapped;
        if (i > 0) {
            LSD_CHECK(ctx, cudaEventRecord(ctx->groupEvent, ctx->stream));
            LSD_CHECK(c0, cudaStreamWaitEvent(c0->stream, ctx->groupEvent, 0));
        }
    }
    *failed = 0;
    // the descriptors go through the launching context's pinned staging: the previous group launch that read it has completed
    // (its results were waited for), and the copy is ordered before this launch on the same stream
    LSD_CHECK(c0, cudaMemcpyAsync(c0->dGroupSegs, h, n * sizeof(TrackGroupSeg), cudaMemcpyHostToDevice, c0->stream));
    const TrackGroupSeg* dSegs = (const TrackGroupSeg*)c0->dGroupSegs;
    void* args[] = { (void*)&dSegs, (void*)&Gs, (void*)&Gv };
    if (c0->profileTrackKernel) cudaEventRecord(c0->kBegin, c0->stream);
    LSD_CHECK(c0, launchCooperative((const void*)k_track_persistent_group, n * Gs, c0->stream, args));
    c0->launches++;
    if (c0->profileTrackKernel) cudaEventRecord(c0->kEnd, c0->stream);
    LSD_CHECK(c0, cudaEventRecord(c0->groupEvent, c0->stream));
    for (int i = 1; i < n; i++) {
        *failed = i;
        LSD_CHECK(ctxs[i], cudaStreamWaitEvent(ctxs[i]->stream, c0->groupEvent, 0));
    }

    double bytes = 0;
    for (int i = 0; i < n; i++) {
        lsdgpu_ctx* ctx = ctxs[i];
        frs[i]->hasGoodMask = true;
        memset(&outs[i], 0, sizeof(outs[i]));
        *failed = i;
        const int r = waitTrackState(ctx, c0->stream);
        if (r) return r;
        bytes += trackAlgorithmicBytes(ctx, (const TrackState*)ctx->hTrackState);
        trackLaunchDone(ctx, (unsigned int)Gs, &outs[i]);                       // this segment's barrier counts Gs CTAs per pass
    }
    if (c0->profileTrackKernel) {            // one launch for the whole group, accounted on the launching context
        c0->trackKernelBytes += bytes;
        c0->trackProfilePending = true;
    }
    return 0;
}
