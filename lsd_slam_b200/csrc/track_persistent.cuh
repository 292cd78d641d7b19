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
#include "track_common.cuh"

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
