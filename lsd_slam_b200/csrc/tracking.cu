// tracking.cu -- SE3 tracking entry points of the C ABI (include/lsdgpu.h): the stand-alone evaluation, the host LM loop of
// mode 0 and its sharded form, the persistent tracker of mode 1 and its group launch over several contexts, and the fused
// track-and-map calls.  Host-side control flow mirrors SE3Tracker::trackFrame (Tracking/SE3Tracker.cpp:280-486).
#include "internal.cuh"
#include "track_persistent.cuh"

#include <algorithm>
#include <atomic>
#include <functional>
#include <stdlib.h>

// CTA-level reduction of all channels: warp shuffles, then one smem stage.  Result valid in warp 0, lane c.
template <int NWARPS>
__device__ __forceinline__ void blockReduceChannels(PointAcc& acc, float (*sm)[EV_NCH], float* blockRow)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < EV_NCH; c++) {
        float v = acc.v[c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) sm[warp][c] = v;
    }
    __syncthreads();
    if (threadIdx.x < EV_NCH) {
        float s = 0.f;
#pragma unroll
        for (int wi = 0; wi < NWARPS; wi++) s += sm[wi][threadIdx.x];
        blockRow[threadIdx.x] = s;
    }
}


// Stand-alone evaluation kernel (one launch per LM evaluation; mode-0 tracker and the parity hook).
__global__ void __launch_bounds__(EVAL_THREADS) k_se3_eval(EvalLevel L, EvalPose P, EvalConsts C,
                                                           float* __restrict__ partials, unsigned int* counter,
                                                           float* __restrict__ out)
{
    __shared__ float sm[EVAL_THREADS / 32][EV_NCH];
    __shared__ bool isLast;
    PointAcc acc;
#pragma unroll
    for (int c = 0; c < EV_NCH; c++) acc.v[c] = 0.f;

    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int w = L.w, h = L.h;
    if (i < w * h) {
        const int x = i % w, y = i / w;
        if (x >= 1 && x < w - 1 && y >= 1 && y < h - 1 && (L.nShards <= 1 || ((i >> 5) % L.nShards) == L.shard)) {
            const float idepth = L.kfIdepth[i], var = L.kfVar[i];
            if (!(var <= 0 || idepth == 0)) {                     // TrackingReference.cpp:133
                const float sc = 1.0f / idepth;                   // :135
                const float px = sc * (L.fxi * x + L.cxi), py = sc * (L.fyi * y + L.cyi), pz = sc * 1;
                const float4* fg = L.frameGrad;
                auto tap = [fg, w](float u, float v, float& o0, float& o1, float& o2) { interp43(fg, u, v, w, o0, o1, o2); };
                int good = evalPoint(px, py, pz, L.kfColor[i], var, P, C, L.fx, L.fy, L.cx, L.cy, w, h, tap, acc);
                if (L.goodMask) L.goodMask[i] = (uint8_t)good;
            }
        }
    }
    blockReduceChannels<EVAL_THREADS / 32>(acc, sm, partials + (size_t)blockIdx.x * EV_NCH);

    // last-CTA-done: deterministic cross-block sum in block order
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned int t = atomicAdd(counter, 1u);
        isLast = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (isLast) {
        __threadfence();
        // EV_NCH channels x 4 partial lanes each (fixed interleave), then a fixed 4-way combine
        const int c = threadIdx.x >> 2, part = threadIdx.x & 3;
        if (c < EV_NCH) {
            double s = 0.0;
            for (int b = part; b < (int)gridDim.x; b += 4) s += (double)__ldcg(partials + (size_t)b * EV_NCH + c);
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            if (part == 0) out[c] = (float)s;
        }
        if (threadIdx.x == 0) *counter = 0;
    }
}

// SE3Tracker's public fields after trackFrame (SE3Tracker.cpp:453-485) from the final referenceToFrame and the statistics of
// the last evaluated pose; mode 0 (trackHostLM) and mode 1 (translateTrackState) both end here.  The call counters are the caller's.
static void finishTrackResult(const lsdgpu_ctx* ctx, const lsd::SE3<float>& referenceToFrame, float pointUsage, float goodCount,
                              float badCount, float meanRes, float lastResidual, float affine_a, float affine_b, bool diverged,
                              lsdgpu_track_result* out)
{
    out->pointUsage = pointUsage; out->lastGoodCount = goodCount; out->lastBadCount = badCount;
    out->lastMeanRes = meanRes;
    out->affineEstimation_a = affine_a; out->affineEstimation_b = affine_b;
    if (diverged) {
        out->frameToRef_qt[3] = 1;
        out->diverged = 1; out->trackingWasGood = 0;
        return;
    }
    const int W = ctx->w, H = ctx->h;
    out->lastResidual = lastResidual;
    out->trackingWasGood = goodCount / ((W >> SE3TRACKING_MIN_LEVEL) * (H >> SE3TRACKING_MIN_LEVEL)) > 0.04f
                           && goodCount / (goodCount + badCount) > 0.5f;                                  // :475-477
    out->initialTrackedResidual = out->lastResidual / out->pointUsage;                                    // :482
    lsd::SE3<double> f2r = lsd::se3Cast<double>(lsd::se3Inverse(referenceToFrame));                        // :483-485
    for (int i = 0; i < 4; i++) out->frameToRef_qt[i] = f2r.q[i];
    for (int i = 0; i < 3; i++) out->frameToRef_qt[4 + i] = f2r.t[i];
}

cudaError_t trackPersistentSetup(lsdgpu_ctx* ctx)
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
    for (int l = 0; l < LSD_LEVELS; l++) {
        out->numCalcResidualCalls[l] = hOut->numCalcResidualCalls[l];
        out->numCalcWarpUpdateCalls[l] = hOut->numCalcWarpUpdateCalls[l];
    }
    lsd::SE3<float> T;
    for (int i = 0; i < 4; i++) T.q[i] = hOut->refToFrame[i];
    for (int i = 0; i < 3; i++) T.t[i] = hOut->refToFrame[4 + i];
    finishTrackResult(ctx, T, hOut->pointUsage, hOut->goodCount, hOut->badCount, hOut->meanRes, hOut->lastResidual, hOut->affine_a,
                      hOut->affine_b, hOut->diverged != 0, out);
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

// Frame::refPixelWasGood(): created on first use, initialised to true (DataStructures/Frame.h:421-437)
static int ensureGoodMask(lsdgpu_ctx* ctx, FrameSlot* fr)
{
    if (fr->hasGoodMask) return 0;
    LSD_CHECK(ctx, cudaMemsetAsync(fr->goodMask, 1, ((size_t)ctx->w * ctx->h) / 4, ctx->stream));
    fr->hasGoodMask = true;
    return 0;
}

static void fillEvalLevel(lsdgpu_ctx* ctx, FrameSlot* kf, FrameSlot* fr, int level, bool writeMask, EvalLevel& L)
{
    const LevelCam& c = ctx->cam[level];
    L.kfIdepth = kf->idepth[level]; L.kfVar = kf->idepthVar[level]; L.kfColor = kf->image[level];
    L.frameGrad = fr->grad[level];
    L.goodMask = writeMask ? fr->goodMask : nullptr;
    L.w = c.w; L.h = c.h;
    L.fx = c.fx; L.fy = c.fy; L.cx = c.cx; L.cy = c.cy;
    L.fxi = c.fxi; L.fyi = c.fyi; L.cxi = c.cxi; L.cyi = c.cyi;
    L.shard = 0; L.nShards = 1;
}

// one evaluation launch + readback of the EV_NCH sums into ctx->hEvOut (synchronous)
static int runEval(lsdgpu_ctx* ctx, const EvalLevel& L, const lsd::SE3<float>& refToFrame, float a, float b,
                   const lsdgpu_track_settings* s)
{
    EvalPose P;
    lsd::quatToMatrix(refToFrame.q, P.R);
    P.t[0] = refToFrame.t[0]; P.t[1] = refToFrame.t[1]; P.t[2] = refToFrame.t[2];
    P.a = a; P.b = b;
    EvalConsts C;
    C.cameraPixelNoise2 = ctx->g.cameraPixelNoise2; C.var_weight = s->var_weight; C.huber_half = s->huber_d / 2;
    const int nBlocks = divUp(L.w * L.h, EVAL_THREADS);
    if (ctx->profileTrackKernel) cudaEventRecord(ctx->kBegin, ctx->stream);
    // last-block counter of its own (word 16): evCounter[0] is the persistent tracker's monotonic barrier counter, which must
    // never be reset or counted on by anybody else (mode-1 and mode-0 / parity-hook calls interleave on one context)
    k_se3_eval<<<nBlocks, EVAL_THREADS, 0, ctx->stream>>>(L, P, C, ctx->evPartials, ctx->evCounter + 16, ctx->dEvOut);
    LAUNCH(ctx);
    if (ctx->profileTrackKernel) cudaEventRecord(ctx->kEnd, ctx->stream);
    LSD_CHECK(ctx, cudaGetLastError());
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->hEvOut, ctx->dEvOut, EV_NCH * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->profileTrackKernel) {
        float ms = 0;
        cudaEventElapsedTime(&ms, ctx->kBegin, ctx->kEnd);
        ctx->trackKernelMs += ms;
        ctx->trackKernelLaunches++;
        // B_fused(l) = 12 B/px keyframe planes + 16 B/px frame gradients (+1 B/px mask on L1) + EV_NCH*4
        ctx->trackKernelBytes += (double)L.w * L.h * (12.0 + 16.0 + (L.goodMask ? 1.0 : 0.0)) + EV_NCH * 4.0;
    }
    return 0;
}

extern "C" int lsdgpu_se3_eval(lsdgpu_ctx* ctx, int kf_id, int frame_id, int level, const float refToFrame_qt[7],
                               float affine_a, float affine_b, const lsdgpu_track_settings* s, int write_good_mask,
                               lsdgpu_eval_result* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    FrameSlot* fr = findSlot(ctx, frame_id);
    if (!kf || !fr) return failMissing(ctx, kf ? frame_id : kf_id, "unknown frame id");
    if (level < 0 || level >= LSD_LEVELS) return lsd_fail(ctx, "bad level");
    int r = ensureIdepthPyramid(ctx, kf);
    if (r) return r;
    lsdgpu_track_settings ds;
    if (!s) { lsdgpu_default_track_settings(&ds); s = &ds; }
    EvalLevel L;
    const bool wm = write_good_mask && level == SE3TRACKING_MIN_LEVEL;
    if (wm) { r = ensureGoodMask(ctx, fr); if (r) return r; }
    fillEvalLevel(ctx, kf, fr, level, wm, L);
    lsd::SE3<float> T;
    for (int i = 0; i < 4; i++) T.q[i] = refToFrame_qt[i];
    for (int i = 0; i < 3; i++) T.t[i] = refToFrame_qt[4 + i];
    r = runEval(ctx, L, T, affine_a, affine_b, s);
    if (r) return r;
    evalFinish(ctx->hEvOut, out);
    return 0;
}

// SE3Tracker::trackFrame with the LM loop on the host (mode 0): a line-by-line mirror of SE3Tracker.cpp:280-486
static int trackHostLM(lsdgpu_ctx* ctx, FrameSlot* kf, FrameSlot* fr, const double init_qt[7],
                       const lsdgpu_track_settings* st, lsdgpu_track_result* out,
                       int shard = 0, int nShards = 1, lsdgpu_allreduce_fn allreduce = nullptr, void* user = nullptr)
{
    memset(out, 0, sizeof(*out));
    bool diverged = false;
    float affine_a = 1, affine_b = 0;
    lsd::SE3<double> init;
    for (int i = 0; i < 4; i++) init.q[i] = init_qt[i];
    for (int i = 0; i < 3; i++) init.t[i] = init_qt[4 + i];
    lsd::SE3<float> referenceToFrame = lsd::se3Cast<float>(lsd::se3Inverse(init));      // :306
    lsdgpu_eval_result ev, lsq;
    memset(&ev, 0, sizeof(ev));
    float last_residual = 0;
    const int W = ctx->w, H = ctx->h;
    { int r0 = ensureGoodMask(ctx, fr); if (r0) return r0; }

    for (int lvl = SE3TRACKING_MAX_LEVEL - 1; lvl >= SE3TRACKING_MIN_LEVEL && !diverged; lvl--) {
        EvalLevel L;
        fillEvalLevel(ctx, kf, fr, lvl, lvl == SE3TRACKING_MIN_LEVEL, L);
        L.shard = shard; L.nShards = nShards;
        int r = runEval(ctx, L, referenceToFrame, affine_a, affine_b, st);
        if (r) return r;
        if (allreduce) allreduce(user, ctx->hEvOut, EV_NCH);
        evalFinish(ctx->hEvOut, &ev);
        if (ev.warpedSize < 0.01f * (W >> lvl) * (H >> lvl)) { diverged = true; break; }   // :324-329
        if (ctx->g.useAffineLightningEstimation) { affine_a = ev.affine_a_lastIt; affine_b = ev.affine_b_lastIt; }
        // NB: the weights of calcWeightsAndResidual (:336) do not depend on the affine parameters just
        // updated (the residual buffer was filled before), so one fused pass yields lastErr and ls
        float lastErr = ev.meanWeightedRes;
        lsq = ev;
        out->numCalcResidualCalls[lvl]++;
        float LM_lambda = st->lambdaInitial[lvl];

        for (int iteration = 0; iteration < st->maxItsPerLvl[lvl] && !diverged; iteration++) {
            out->numCalcWarpUpdateCalls[lvl]++;         // calculateWarpUpdate(ls): lsq already holds it
            int incTry = 0;
            while (true) {
                float b[6], A[36], inc[6];
                for (int i = 0; i < 6; i++) b[i] = -lsq.b[i];
                memcpy(A, lsq.A, sizeof(A));
                for (int i = 0; i < 6; i++) A[i * 6 + i] *= 1 + LM_lambda;
                lsd::ldlt6Solve(A, b, inc);
                incTry++;
                lsd::SE3<float> new_referenceToFrame = lsd::se3Mul(lsd::se3Exp(inc), referenceToFrame);   // :363
                r = runEval(ctx, L, new_referenceToFrame, affine_a, affine_b, st);
                if (r) return r;
                if (allreduce) allreduce(user, ctx->hEvOut, EV_NCH);
                evalFinish(ctx->hEvOut, &ev);
                if (ev.warpedSize < 0.01f * (W >> lvl) * (H >> lvl)) { diverged = true; break; }
                float error = ev.meanWeightedRes;
                out->numCalcResidualCalls[lvl]++;
                if (error < lastErr) {
                    referenceToFrame = new_referenceToFrame;
                    if (ctx->g.useAffineLightningEstimation) { affine_a = ev.affine_a_lastIt; affine_b = ev.affine_b_lastIt; }
                    if (error / lastErr > st->convergenceEps[lvl]) iteration = st->maxItsPerLvl[lvl];
                    last_residual = lastErr = error;
                    lsq = ev;                         // buffers now belong to the accepted pose
                    if (LM_lambda <= 0.2) LM_lambda = 0;
                    else LM_lambda *= st->lambdaSuccessFac;
                    break;
                } else {
                    float dot = 0;
                    for (int i = 0; i < 6; i++) dot += inc[i] * inc[i];
                    if (!(dot > st->stepSizeMin[lvl])) { iteration = st->maxItsPerLvl[lvl]; break; }
                    if (LM_lambda == 0) LM_lambda = 0.2;
                    else LM_lambda *= pow((double)st->lambdaFailFac, incTry);
                }
            }
        }
    }
    finishTrackResult(ctx, referenceToFrame, ev.pointUsage, ev.goodCount, ev.badCount, ev.meanRes, last_residual, affine_a, affine_b,
                      diverged, out);
    return 0;
}

// `s`, or for a null `s` the main tracker's settings: the defaults without iterations on level 4 (SlamSystem.cpp:80-81)
static const lsdgpu_track_settings* trackSettingsOrDefault(const lsdgpu_track_settings* s, lsdgpu_track_settings& ds)
{
    if (s) return s;
    lsdgpu_default_track_settings(&ds);
    ds.maxItsPerLvl[4] = 0;
    return &ds;
}

// the Frame side effects of a tracking that did not diverge (SE3Tracker.cpp:479-484)
static void applyTrackedFrame(FrameSlot* kf, FrameSlot* fr, const lsdgpu_track_result* out)
{
    if (out->diverged) return;
    if (out->trackingWasGood) kf->numFramesTrackedOnThis++;                   // :479-480
    fr->initialTrackedResidual = out->initialTrackedResidual;                 // :482
    for (int i = 0; i < 7; i++) fr->thisToParent[i] = out->frameToRef_qt[i];  // :483 sim3FromSE3(.., 1)
    fr->thisToParent[7] = 1.0;
    fr->parentId = kf->id;                                                    // :484
}

extern "C" int lsdgpu_se3_track(lsdgpu_ctx* ctx, int kf_id, int frame_id, const double init_qt[7],
                                const lsdgpu_track_settings* s, int mode, lsdgpu_track_result* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    FrameSlot* fr = findSlot(ctx, frame_id);
    if (!kf || !fr) return failMissing(ctx, kf ? frame_id : kf_id, "unknown frame id");
    int r = ensureIdepthPyramid(ctx, kf);      // reference->makePointCloud(lvl), SE3Tracker.cpp:321
    if (r) return r;
    lsdgpu_track_settings ds;
    s = trackSettingsOrDefault(s, ds);
    if (mode == 1) r = trackPersistent(ctx, kf, fr, init_qt, s, out);
    else r = trackHostLM(ctx, kf, fr, init_qt, s, out);
    if (r) return r;
    applyTrackedFrame(kf, fr, out);
    return 0;
}

static_assert(LSDGPU_EVAL_NSUMS == EV_NCH, "ABI constant out of sync with the kernel's channel count");

extern "C" int lsdgpu_se3_track_sharded(lsdgpu_ctx* ctx, int kf_id, int frame_id, const double init_qt[7],
                                        const lsdgpu_track_settings* s, int shard, int n_shards,
                                        lsdgpu_allreduce_fn allreduce, void* user, lsdgpu_track_result* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    FrameSlot* fr = findSlot(ctx, frame_id);
    if (!kf || !fr) return failMissing(ctx, kf ? frame_id : kf_id, "unknown frame id");
    if (n_shards < 1 || shard < 0 || shard >= n_shards) return lsd_fail(ctx, "bad shard");
    if (n_shards > 1 && !allreduce) return lsd_fail(ctx, "sharded tracking needs an all-reduce callback");
    int r = ensureIdepthPyramid(ctx, kf);
    if (r) return r;
    lsdgpu_track_settings ds;
    r = trackHostLM(ctx, kf, fr, init_qt, trackSettingsOrDefault(s, ds), out, shard, n_shards, allreduce, user);
    if (r) return r;
    applyTrackedFrame(kf, fr, out);
    return 0;
}

extern "C" int lsdgpu_track_kernel_stats(lsdgpu_ctx* ctx, int reset, double* ms, long long* launches, double* bytes)
{ LSD_LOCK(ctx);
    flushTrackProfile(ctx);
    if (ms) *ms = ctx->trackKernelMs;
    if (launches) *launches = ctx->trackKernelLaunches;
    if (bytes) *bytes = ctx->trackKernelBytes;
    if (reset == 1) { ctx->trackKernelMs = 0; ctx->trackKernelLaunches = 0; ctx->trackKernelBytes = 0; ctx->profileTrackKernel = true; }
    if (reset == 2) ctx->profileTrackKernel = false;
    return 0;
}

extern "C" int lsdgpu_track_and_map(lsdgpu_ctx* ctx, int kf_id, int frame_id, const uint8_t* gray, int stage_index,
                                    const double init_qt[7], const lsdgpu_track_settings* s, int mode,
                                    int keyframe_change, lsdgpu_track_result* out, double new_qts[8])
{ LSD_LOCK(ctx);
    if (findMinimized(ctx, kf_id)) return failMissing(ctx, kf_id, "unknown keyframe id");      // before the frame is built
    int r = gray ? lsdgpu_frame_upload_u8(ctx, frame_id, gray) : lsdgpu_frame_from_stage(ctx, frame_id, stage_index);
    if (r) return r;
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return lsd_fail(ctx, "unknown keyframe id");
    if (kf->depthHasBeenUpdatedFlag) { r = lsdgpu_ref_import(ctx, kf_id); if (r) return r; }     // SlamSystem.cpp:907-912
    r = lsdgpu_se3_track(ctx, kf_id, frame_id, init_qt, s, mode, out);
    if (r) return r;
    if (out->diverged) return 0;                 // the caller decides (relocalisation is out of scope)
    if (keyframe_change) {
        r = lsdgpu_depth_finalize_keyframe(ctx);
        if (r) return r;
        return lsdgpu_depth_create_keyframe(ctx, frame_id, new_qts);
    }
    r = lsdgpu_depth_update_keyframe(ctx, &frame_id, 1);
    if (r) return r;
    return lsdgpu_frame_clear_good_mask(ctx, frame_id);
}

// ------------------------------------------------------------------------------------------------------
// several streams per GPU: one tracking launch for the frames of n contexts
// ------------------------------------------------------------------------------------------------------
// the message goes to every context of the group (each one's own lock is taken again: recursive)
static int groupFail(int n, const lsdgpu_group_step* steps, int step, const char* msg, int rc = -2)
{
    char b[600];
    if (step >= 0) snprintf(b, sizeof(b), "track_and_map_group: step %d: %s", step, msg);
    else snprintf(b, sizeof(b), "track_and_map_group: %s", msg);
    for (int i = 0; i < n; i++)
        if (steps[i].ctx) { CtxLock l(steps[i].ctx); steps[i].ctx->err = b; }
    return rc;
}
// an entry point called for step `step` failed and set its context's message: hand it to the whole group
static int groupPropagate(int n, const lsdgpu_group_step* steps, int step, int rc)
{
    const std::string m = steps[step].ctx->err;
    return groupFail(n, steps, step, m.c_str(), rc);
}

extern "C" int lsdgpu_track_and_map_group(int n, const lsdgpu_group_step* steps, lsdgpu_track_result* results, double* new_qts)
{
    if (!steps || n < 1) return -2;
    if (n > TP_MAX_GROUP) return groupFail(n, steps, -1, "the number of steps must be 1..8");
    for (int i = 0; i < n; i++)
        if (!steps[i].ctx) return groupFail(n, steps, i, "null context");
    if (!results) return groupFail(n, steps, -1, "null result array");
    for (int i = 1; i < n; i++)
        for (int j = 0; j < i; j++)
            if (steps[i].ctx == steps[j].ctx) return groupFail(n, steps, i, "the same context as an earlier step");
    // every context's lock for the whole call, taken in ascending address order: two threads issuing overlapping groups cannot deadlock
    lsdgpu_ctx* order[TP_MAX_GROUP];
    for (int i = 0; i < n; i++) order[i] = steps[i].ctx;
    std::sort(order, order + n, std::less<lsdgpu_ctx*>());
    std::unique_lock<std::recursive_mutex> locks[TP_MAX_GROUP];
    for (int i = 0; i < n; i++) locks[i] = std::unique_lock<std::recursive_mutex>(order[i]->mu);

    lsdgpu_ctx* c0 = steps[0].ctx;
    for (int i = 0; i < n; i++) {
        const lsdgpu_ctx* c = steps[i].ctx;
        if (c->device != c0->device) return groupFail(n, steps, i, "context is on another device than step 0's");
        if (c->w != c0->w || c->h != c0->h) return groupFail(n, steps, i, "context size differs from step 0's");
        if (c->nRanks > 1) return groupFail(n, steps, i, "context is peer-attached (a sharded stream cannot be grouped)");
        if (!findSlot(steps[i].ctx, steps[i].kf_id)) {
            if (findMinimized(steps[i].ctx, steps[i].kf_id)) return groupFail(n, steps, i, ("keyframe " + std::to_string(steps[i].kf_id) + " is minimized").c_str());
            return groupFail(n, steps, i, "unknown frame id (keyframe)");
        }
        if (findMinimized(steps[i].ctx, steps[i].frame_id)) return groupFail(n, steps, i, ("frame " + std::to_string(steps[i].frame_id) + " is minimized").c_str());
    }
    if (cudaSetDevice(c0->device) != cudaSuccess) return groupFail(n, steps, -1, "cudaSetDevice failed", -1);

    // 1. per step, on its own stream: Frame construction, importFrame if the keyframe's depth changed (SlamSystem.cpp:907-912)
    lsdgpu_ctx* ctxs[TP_MAX_GROUP];
    FrameSlot* kfs[TP_MAX_GROUP];
    FrameSlot* frs[TP_MAX_GROUP];
    const double* inits[TP_MAX_GROUP];
    const lsdgpu_track_settings* sts[TP_MAX_GROUP];
    lsdgpu_track_settings ds[TP_MAX_GROUP];
    for (int i = 0; i < n; i++) {
        const lsdgpu_group_step& st = steps[i];
        lsdgpu_ctx* ctx = st.ctx;
        ctxs[i] = ctx;
        int r = st.gray ? lsdgpu_frame_upload_u8(ctx, st.frame_id, st.gray) : lsdgpu_frame_from_stage(ctx, st.frame_id, st.stage_index);
        if (r) return groupPropagate(n, steps, i, r);
        kfs[i] = findSlot(ctx, st.kf_id);
        frs[i] = findSlot(ctx, st.frame_id);
        if (!kfs[i] || !frs[i]) return groupFail(n, steps, i, "unknown frame id");
        if (kfs[i]->depthHasBeenUpdatedFlag) {
            r = lsdgpu_ref_import(ctx, st.kf_id);
            if (r) return groupPropagate(n, steps, i, r);
        }
        r = ensureIdepthPyramid(ctx, kfs[i]);                // as lsdgpu_se3_track
        if (r) return groupPropagate(n, steps, i, r);
        inits[i] = st.frameToRef_init_qt;
        sts[i] = trackSettingsOrDefault(st.settings, ds[i]);
    }
    // 2-5. one launch on steps[0]'s stream for all the frames
    int failed = 0;
    int r = trackPersistentGroup(n, ctxs, kfs, frs, inits, sts, results, &failed);
    if (r) return groupPropagate(n, steps, failed, r);
    for (int i = 0; i < n; i++) applyTrackedFrame(kfs[i], frs[i], &results[i]);    // as lsdgpu_se3_track
    // 6. mapping, each step on its own stream; a diverged step maps nothing.  The contexts are independent, so the order across
    // steps is free: the keyframe changes, whose createKeyFrame waits for its stream, go last so that the updates of the other
    // streams are already in flight.
    for (int pass = 0; pass < 2; pass++)
        for (int i = 0; i < n; i++) {
            const lsdgpu_group_step& st = steps[i];
            if (results[i].diverged || (st.keyframe_change != 0) != (pass == 1)) continue;
            if (st.keyframe_change) {
                r = lsdgpu_depth_finalize_keyframe(st.ctx);
                if (!r) r = lsdgpu_depth_create_keyframe(st.ctx, st.frame_id, new_qts ? new_qts + 8 * i : nullptr);
            } else {
                r = lsdgpu_depth_update_keyframe(st.ctx, &st.frame_id, 1);
                if (!r) r = lsdgpu_frame_clear_good_mask(st.ctx, st.frame_id);
            }
            if (r) return groupPropagate(n, steps, i, r);
        }
    return 0;
}
