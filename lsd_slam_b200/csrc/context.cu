// context.cu -- the context of the C ABI (include/lsdgpu.h): creation and its device arena, destruction, errors, globals,
// timers, and the peer mapping of one stream's contexts over several GPUs.
#include "internal.cuh"
#include "track_common.cuh"

#include <new>

extern "C" int lsdgpu_abi_version(void) { return LSDGPU_ABI_VERSION; }

extern "C" void lsdgpu_default_globals(lsdgpu_globals* g)
{
    g->minUseGrad = 5; g->cameraPixelNoise2 = 4 * 4; g->depthSmoothingFactor = 1;
    g->allowNegativeIdepths = 1; g->useSubpixelStereo = 1; g->useAffineLightningEstimation = 1;
}

extern "C" void lsdgpu_default_track_settings(lsdgpu_track_settings* s)
{
    static const int maxIterations[6] = { 5, 20, 50, 100, 100, 100 };
    s->lambdaSuccessFac = 0.5f; s->lambdaFailFac = 2.0f;
    for (int l = 0; l < LSD_LEVELS; l++) {
        s->lambdaInitial[l] = 0; s->stepSizeMin[l] = 1e-8f; s->convergenceEps[l] = 0.999f;
        s->maxItsPerLvl[l] = maxIterations[l];
    }
    s->var_weight = 1.0f; s->huber_d = 3;
}

static void setupCams(lsdgpu_ctx* ctx, const float K[9])
{   // Frame::initialize, DataStructures/Frame.cpp:403-459
    LevelCam& c0 = ctx->cam[0];
    memcpy(c0.K, K, 36);
    c0.w = ctx->w; c0.h = ctx->h;
    c0.fx = K[0]; c0.fy = K[4]; c0.cx = K[2]; c0.cy = K[5];
    lsd::mat3Inverse(c0.K, c0.KInv);
    c0.fxi = c0.KInv[0]; c0.fyi = c0.KInv[4]; c0.cxi = c0.KInv[2]; c0.cyi = c0.KInv[5];
    for (int l = 1; l < LSD_LEVELS; l++) {
        LevelCam& c = ctx->cam[l];
        c.w = ctx->w >> l; c.h = ctx->h >> l;
        c.fx = (float)(ctx->cam[l - 1].fx * 0.5);
        c.fy = (float)(ctx->cam[l - 1].fy * 0.5);
        c.cx = (float)((c0.cx + 0.5) / ((int)1 << l) - 0.5);
        c.cy = (float)((c0.cy + 0.5) / ((int)1 << l) - 0.5);
        float Kl[9] = { c.fx, 0.f, c.cx, 0.f, c.fy, c.cy, 0.f, 0.f, 1.f };
        memcpy(c.K, Kl, 36);
        lsd::mat3Inverse(c.K, c.KInv);
        c.fxi = c.KInv[0]; c.fyi = c.KInv[4]; c.cxi = c.KInv[2]; c.cyi = c.KInv[5];
    }
}

// Every buffer of the context's arena, in layout order, each at a 256-byte boundary.  With a null `base` only the size is
// measured (the pointers stay null); on the allocation the same list carves it.  Peer-attached ranks address each other's
// buffers by their offset in the arena (lsdgpu_peer_attach), so the layout must depend on nothing but the context's size.
static size_t carveArena(lsdgpu_ctx* ctx, char* base)
{
    size_t used = 0;
    auto take = [&](size_t bytes) { char* r = base ? base + used : nullptr; used += alignUp(bytes, 256); return r; };
    const size_t n0 = (size_t)ctx->w * ctx->h;
    const int maxBlocks = divUp((int)n0, EVAL_THREADS) + 8;
    const int seqRuns = divUp((int)n0, SEQ_RUN);
    for (auto& s : ctx->slots) {
        for (int l = 0; l < LSD_LEVELS; l++) {
            size_t n = n0 >> (2 * l);
            s.image[l] = (float*)take(n * 4);
            s.grad[l] = (float4*)take(n * 16);
            s.idepth[l] = (float*)take(n * 4);
            s.idepthVar[l] = (float*)take(n * 4);
        }
        s.maxgrad = (float*)take(n0 * 4);
        s.goodMask = (uint8_t*)take(n0 / 4);
    }
    ctx->cur.hf = (float4*)take(n0 * 16); ctx->cur.hi = (int4*)take(n0 * 16);
    ctx->oth.hf = (float4*)take(n0 * 16); ctx->oth.hi = (int4*)take(n0 * 16);
    ctx->integral = (int*)take(n0 * 4);
    ctx->propHead = (int*)take(n0 * 4);
    ctx->propNext = (int*)take(n0 * 4);
    ctx->propVal = (float4*)take(n0 * 16);
    ctx->evPartials = (float*)take((size_t)maxBlocks * EV_NCH * 4 + 65536);   // also holds the 2 x 160 x 192 B exchange rows of mode 1
    ctx->evCounter = (unsigned int*)take(256);
    ctx->trkSync = (unsigned int*)take(TP_SYNC_WORDS * 4);
    ctx->dEvOut = (float*)take(EV_NCH * 4);
    ctx->dStageU8[0] = (uint8_t*)take(n0);
    ctx->dStageU8[1] = (uint8_t*)take(n0);
    for (auto& s : ctx->slots) {
        s.dStats = (double*)take(64);
        s.permaPC = (float4*)take((n0 >> 8) * 16);
        s.permaVar = (float*)take((n0 >> 8) * 4);
        s.reactIdepth = (float*)take(n0 * 4);
        s.reactVar = (float*)take(n0 * 4);
        s.reactValidity = (uint8_t*)take(n0);
    }
    ctx->dPacked = (uint32_t*)take(n0 * 12);
    ctx->dPermaItems = take(LSD_MAX_PERMA_BATCH * sizeof(PermaItem));
    ctx->dPermaResults = take(LSD_MAX_PERMA_BATCH * sizeof(PermaResult));
    ctx->dSim3Items = take(S3_MAX_BATCH * sizeof(Sim3Item));
    ctx->dSim3Outs = take(S3_MAX_BATCH * sizeof(Sim3Out));
    ctx->dStageF = (float*)take(n0 * 32);
    ctx->dScalars = (double*)take((size_t)maxBlocks * 2 * 8 + 64);
    ctx->seqTable = (int2*)take((size_t)seqRuns * SEQ_NBIN * sizeof(int2));
    ctx->seqFlags = (unsigned char*)take((size_t)seqRuns);
    ctx->seqCounts = (int*)take((size_t)seqRuns * 4);
    ctx->dLastMask = (uint8_t*)take(n0 / 4);
    ctx->dGroupSegs = take(TP_MAX_GROUP * sizeof(TrackGroupSeg));
    ctx->rndTab = (uint32_t*)take((size_t)RND_TYPES * RND_TYPE_WORDS * 4);
    ctx->rndTiles = (int*)take(((size_t)divUp((int)n0, RND_TILE) + 1) * 4);
    ctx->rndOut = (uint32_t*)take(4 + RND_ROW * 4);
    return used;
}

extern "C" int lsdgpu_create(int device, int width, int height, const float K[9], int max_frames, lsdgpu_ctx** out)
{
    if (!out) return -2;
    *out = nullptr;
    if (width <= 0 || height <= 0 || (width % 16) || (height % 16) || max_frames < 2) return -2;   // SlamSystem.cpp:55
    lsdgpu_ctx* ctx = new (std::nothrow) lsdgpu_ctx();
    if (!ctx) return -3;
    *out = ctx;      // returned even on failure so that lsdgpu_last_error can be read
    ctx->device = device; ctx->w = width; ctx->h = height;
    lsdgpu_default_globals(&ctx->g);
    setupCams(ctx, K);
    LSD_CHECK(ctx, cudaSetDevice(device));
    cudaDeviceProp prop;
    LSD_CHECK(ctx, cudaGetDeviceProperties(&prop, device));
    ctx->smCount = prop.multiProcessorCount;
    LSD_CHECK(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));

    ctx->slots.resize(max_frames);
    for (auto& s : ctx->slots) {
        memset(s.thisToParent, 0, sizeof(s.thisToParent));
        s.thisToParent[3] = 1; s.thisToParent[7] = 1;
    }
    ctx->arenaBytes = carveArena(ctx, nullptr);
    LSD_CHECK(ctx, cudaMalloc((void**)&ctx->arena, ctx->arenaBytes));
    LSD_CHECK(ctx, cudaMemsetAsync(ctx->arena, 0, ctx->arenaBytes, ctx->stream));
    carveArena(ctx, ctx->arena);
    const size_t n0 = (size_t)width * height;

    LSD_CHECK(ctx, cudaHostAlloc((void**)&ctx->hEvOut, EV_NCH * 4, cudaHostAllocDefault));
    for (int i = 0; i < 2; i++) {
        LSD_CHECK(ctx, cudaHostAlloc((void**)&ctx->hStage[i], n0, cudaHostAllocDefault));
        LSD_CHECK(ctx, cudaEventCreateWithFlags(&ctx->stageDone[i], cudaEventDisableTiming));
        LSD_CHECK(ctx, cudaEventRecord(ctx->stageDone[i], ctx->stream));
    }
    LSD_CHECK(ctx, cudaHostAlloc((void**)&ctx->hStageF, n0 * 32, cudaHostAllocDefault));
    LSD_CHECK(ctx, cudaHostAlloc((void**)&ctx->hScalars, 64, cudaHostAllocDefault));
    LSD_CHECK(ctx, cudaHostAlloc(&ctx->hGroupSegs, TP_MAX_GROUP * sizeof(TrackGroupSeg), cudaHostAllocDefault));
    LSD_CHECK(ctx, cudaEventCreateWithFlags(&ctx->groupEvent, cudaEventDisableTiming));
    LSD_CHECK(ctx, cudaEventCreateWithFlags(&ctx->callerIn, cudaEventDisableTiming));
    LSD_CHECK(ctx, cudaEventCreateWithFlags(&ctx->callerOut, cudaEventDisableTiming));
    // the tracker writes its result block straight into mapped pinned memory (no D2H copy on the path)
    LSD_CHECK(ctx, cudaHostAlloc((void**)&ctx->hTrackState, sizeof(TrackState), cudaHostAllocMapped));
    // cudaHostAlloc does not clear: a recycled block may still hold the result of a destroyed context, whose doneSeq would satisfy
    // the completion spin of this context's first launches (trackPersistent) before the kernel has written anything
    memset(ctx->hTrackState, 0, sizeof(TrackState));
    memset(ctx->hScalars, 0, 64);
    memset(ctx->hEvOut, 0, EV_NCH * 4);
    LSD_CHECK(ctx, cudaHostGetDevicePointer(&ctx->dTrackStateMapped, ctx->hTrackState, 0));
    for (int i = 0; i < 8; i++) {
        LSD_CHECK(ctx, cudaEventCreate(&ctx->tBegin[i]));
        LSD_CHECK(ctx, cudaEventCreate(&ctx->tEnd[i]));
    }
    LSD_CHECK(ctx, cudaEventCreate(&ctx->kBegin));
    LSD_CHECK(ctx, cudaEventCreate(&ctx->kEnd));
    LSD_CHECK(ctx, trackPersistentSetup(ctx));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

static void peerCloseAll(lsdgpu_ctx* ctx);

extern "C" void lsdgpu_destroy(lsdgpu_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    peerCloseAll(ctx);
    cloudRelease(ctx);
    for (auto& m : ctx->minimized) freeRecord(ctx, m);
    for (cudaMemPool_t p : ctx->pool)
        if (p) { cudaStreamSynchronize(ctx->stream); cudaMemPoolDestroy(p); }
    cudaFree(ctx->arena);
    if (ctx->stageRing) cudaFree(ctx->stageRing);
    if (ctx->dRemapX) cudaFree(ctx->dRemapX);
    if (ctx->dRemapY) cudaFree(ctx->dRemapY);
    if (ctx->dCvMap1) cudaFree(ctx->dCvMap1);
    if (ctx->dCvMap2) cudaFree(ctx->dCvMap2);
    if (ctx->dRaw) cudaFree(ctx->dRaw);
    if (ctx->hRaw) cudaFreeHost(ctx->hRaw);
    cudaFreeHost(ctx->hEvOut); cudaFreeHost(ctx->hStage[0]); cudaFreeHost(ctx->hStage[1]); cudaFreeHost(ctx->hStageF);
    cudaEventDestroy(ctx->stageDone[0]); cudaEventDestroy(ctx->stageDone[1]);
    cudaFreeHost(ctx->hScalars); cudaFreeHost(ctx->hTrackState);
    if (ctx->hGroupSegs) cudaFreeHost(ctx->hGroupSegs);
    if (ctx->groupEvent) cudaEventDestroy(ctx->groupEvent);
    if (ctx->callerIn) cudaEventDestroy(ctx->callerIn);
    if (ctx->callerOut) cudaEventDestroy(ctx->callerOut);
    for (int i = 0; i < 8; i++) { if (ctx->tBegin[i]) cudaEventDestroy(ctx->tBegin[i]); if (ctx->tEnd[i]) cudaEventDestroy(ctx->tEnd[i]); }
    if (ctx->kBegin) cudaEventDestroy(ctx->kBegin);
    if (ctx->kEnd) cudaEventDestroy(ctx->kEnd);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

extern "C" const char* lsdgpu_last_error(const lsdgpu_ctx* ctx) {   // a copy per calling thread: another thread may fail (and overwrite ctx->err) right after this one
    static thread_local std::string mine;
    if (!ctx) return "null context";
    LSD_LOCK(ctx);
    mine = ctx->err;
    return mine.c_str();
}
extern "C" int lsdgpu_set_globals(lsdgpu_ctx* ctx, const lsdgpu_globals* g) { LSD_LOCK(ctx); ctx->g = *g; return 0; }
extern "C" int lsdgpu_get_globals(const lsdgpu_ctx* ctx, lsdgpu_globals* g) { LSD_LOCK(ctx); *g = ctx->g; return 0; }
extern "C" int lsdgpu_synchronize(lsdgpu_ctx* ctx)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}
extern "C" long long lsdgpu_launch_count(const lsdgpu_ctx* ctx) { LSD_LOCK(ctx); return ctx->launches; }

extern "C" int lsdgpu_timer_begin(lsdgpu_ctx* ctx, int slot)
{ LSD_LOCK(ctx);
    if (slot < 0 || slot >= 8) return -2;
    LSD_CHECK(ctx, cudaEventRecord(ctx->tBegin[slot], ctx->stream));
    return 0;
}
extern "C" int lsdgpu_timer_end(lsdgpu_ctx* ctx, int slot)
{ LSD_LOCK(ctx);
    if (slot < 0 || slot >= 8) return -2;
    LSD_CHECK(ctx, cudaEventRecord(ctx->tEnd[slot], ctx->stream));
    return 0;
}
extern "C" int lsdgpu_timer_elapsed_ms(lsdgpu_ctx* ctx, int slot, float* ms)
{ LSD_LOCK(ctx);
    if (slot < 0 || slot >= 8) return -2;
    LSD_CHECK(ctx, cudaEventSynchronize(ctx->tEnd[slot]));
    LSD_CHECK(ctx, cudaEventElapsedTime(ms, ctx->tBegin[slot], ctx->tEnd[slot]));
    return 0;
}
// ------------------------------------------------------------------------------------------------------
// one stream over several GPUs: peer mapping of the contexts' arenas (BASELINE config 5)
// ------------------------------------------------------------------------------------------------------
static_assert(sizeof(cudaIpcMemHandle_t) == LSDGPU_PEER_HANDLE_BYTES, "ABI constant out of sync with cudaIpcMemHandle_t");

extern "C" int lsdgpu_peer_export(lsdgpu_ctx* ctx, void* handle_out)
{ LSD_LOCK(ctx);
    if (!ctx || !handle_out) return lsd_fail(ctx, "peer_export: null argument");
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    LSD_CHECK(ctx, cudaIpcGetMemHandle(&h, ctx->arena));
    memcpy(handle_out, &h, sizeof(h));
    return 0;
}

static void peerCloseAll(lsdgpu_ctx* ctx)
{
    for (int d = 0; d < 8; d++) {
        if (ctx->peerBase[d] && d != ctx->rank) cudaIpcCloseMemHandle(ctx->peerBase[d]);
        ctx->peerBase[d] = nullptr;
    }
    ctx->nRanks = 1; ctx->rank = 0;
}

extern "C" int lsdgpu_peer_attach(lsdgpu_ctx* ctx, int rank, int n_ranks, const void* handles)
{ LSD_LOCK(ctx);
    if (!ctx) return -2;
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (n_ranks < 1 || n_ranks > TP_MAX_RANKS || rank < 0 || rank >= n_ranks) return lsd_fail(ctx, "peer_attach: bad rank / number of ranks");
    if (n_ranks > 1 && !handles) return lsd_fail(ctx, "peer_attach: null handle array");
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    peerCloseAll(ctx);
    if (n_ranks == 1) return 0;
    for (int d = 0; d < n_ranks; d++) {
        if (d == rank) { ctx->peerBase[d] = ctx->arena; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, (const char*)handles + (size_t)d * sizeof(h), sizeof(h));
        void* base = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            ctx->rank = rank;
            peerCloseAll(ctx);
            cudaGetLastError();
            const std::string msg = std::string("peer_attach: cudaIpcOpenMemHandle failed for rank ") + std::to_string(d) + ": " + cudaGetErrorString(e);
            return lsd_fail(ctx, msg.c_str());
        }
        ctx->peerBase[d] = (char*)base;
    }
    ctx->rank = rank; ctx->nRanks = n_ranks;
    // the exchange rows, done slots and the tail counter start from a known state on every rank (the caller synchronises the ranks
    // between attach and the first tracking)
    LSD_CHECK(ctx, cudaMemsetAsync(ctx->trkSync + TP_XCHG_OFFSET, 0, (TP_SYNC_WORDS - TP_XCHG_OFFSET) * sizeof(unsigned int), ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->trkTailBase = 0;
    return 0;
}

extern "C" int lsdgpu_peer_detach(lsdgpu_ctx* ctx)
{ LSD_LOCK(ctx);
    if (!ctx) return -2;
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    peerCloseAll(ctx);
    return 0;
}
