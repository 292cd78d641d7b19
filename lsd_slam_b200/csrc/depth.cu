// depth.cu -- DepthMap entry points of the C ABI (include/lsdgpu.h): observe, regularise, propagate, create / finalize a
// keyframe, re-activation of an old keyframe, and the sequential-sum parity hook.  Host-side control flow mirrors
// DepthMap::updateKeyframe / createKeyFrame / finalizeKeyFrame (DepthEstimation/DepthMap.cpp:1072-1395).
#include "internal.cuh"
#include "depth.cuh"
#include "seqsum.cuh"
#include "rand.cuh"

#include <utility>

static DepthCam depthCam(const lsdgpu_ctx* ctx)
{
    const LevelCam& c = ctx->cam[0];
    DepthCam d;
    d.w = c.w; d.h = c.h; d.fx = c.fx; d.fy = c.fy; d.cx = c.cx; d.cy = c.cy;
    d.fxi = c.fxi; d.fyi = c.fyi; d.cxi = c.cxi; d.cyi = c.cyi;
    return d;
}
static DepthGlobals depthGlobals(const lsdgpu_ctx* ctx)
{
    DepthGlobals g;
    g.minUseGrad = ctx->g.minUseGrad; g.cameraPixelNoise2 = ctx->g.cameraPixelNoise2;
    g.regDistVar = 0.075f * 0.075f * ctx->g.depthSmoothingFactor * ctx->g.depthSmoothingFactor;   // REG_DIST_VAR, settings.h:139
    g.allowNegativeIdepths = ctx->g.allowNegativeIdepths; g.useSubpixelStereo = ctx->g.useSubpixelStereo;
    return g;
}

extern "C" int lsdgpu_depth_reset(lsdgpu_ctx* ctx)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    const size_t n = (size_t)ctx->w * ctx->h;
    // isValid = false everywhere (the int4 plane: isValid, blacklisted, validity, nextId)
    LSD_CHECK(ctx, cudaMemsetAsync(ctx->cur.hi, 0, n * 16, ctx->stream));
    LSD_CHECK(ctx, cudaMemsetAsync(ctx->oth.hi, 0, n * 16, ctx->stream));
    return 0;
}
extern "C" int lsdgpu_depth_is_valid(lsdgpu_ctx* ctx) { LSD_LOCK(ctx); return ctx->activeKf >= 0 ? 1 : 0; }
extern "C" int lsdgpu_depth_invalidate(lsdgpu_ctx* ctx) { LSD_LOCK(ctx); ctx->activeKf = -1; return 0; }
extern "C" int lsdgpu_depth_active_keyframe(lsdgpu_ctx* ctx) { LSD_LOCK(ctx); return ctx->activeKf; }

// Frame::setDepth(currentDepthMap) of the active keyframe
static int setDepthOnKeyframe(lsdgpu_ctx* ctx, FrameSlot* kf)
{
    const int n = ctx->w * ctx->h;
    const int nb = divUp(n, 256);
    PyrPtrs id, var;
    for (int l = 0; l < LSD_LEVELS; l++) { id.l[l] = kf->idepth[l]; var.l[l] = kf->idepthVar[l]; }
    k_set_depth_pyr<<<(ctx->w / 16) * (ctx->h / 16), 256, 0, ctx->stream>>>(ctx->cur, id, var, ctx->w, ctx->h, ctx->dScalars + 8,
                                                                           ctx->evCounter + 48, kf->dStats);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    kf->statsPending = true;
    kf->hasDepth = true; kf->idepthPyrValid = true;          // levels 1..4 were built by the same kernel
    kf->depthHasBeenUpdatedFlag = true;
    return 0;
}

extern "C" int lsdgpu_depth_init_from_gt(lsdgpu_ctx* ctx, int kf_id)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "unknown keyframe id");
    if (!kf->hasDepth) return lsd_fail(ctx, "initializeFromGTDepth: frame has no idepth (call lsdgpu_frame_set_depth_gt)");
    const int n = ctx->w * ctx->h;
    ctx->activeKf = kf_id; ctx->activeKfReactivated = false;
    k_init_from_gt<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->cur, kf->idepth[0], n);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    return setDepthOnKeyframe(ctx, kf);
}

// ---- DepthMap::initializeRandomly, DepthMap.cpp:883-916, with the caller's rand() stream (rand.cuh) ----------------------------
// Three kernels: the draws per tile of RND_TILE pixels, their offsets (a scan), and per tile the jump to its first draw, its
// draws and the cells.  A pixel's draw index is the number of selected pixels before it in raster order.
struct RndEntry {
    int type, deg, winLen;               // winLen: words of the window (deg, 1 for the LCG)
    float minGrad;                       // MIN_ABS_GRAD_CREATE == minUseGrad, util/settings.h:157
    uint32_t W[RND_ROW];                 // the window before the first draw
};

// exclusive prefix of v over the block (NW warps); total = the block's sum
template <int NW>
__device__ __forceinline__ int rndBlockScan(int v, int* sWarp, int& total)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sWarp[wid] = x;
    __syncthreads();
    int off = 0;
    total = 0;
    for (int k = 0; k < NW; k++) {
        const int t = sWarp[k];
        if (k < wid) off += t;
        total += t;
    }
    __syncthreads();
    return off + x - v;
}

// the interior pixels (DepthMap.cpp:892-894) with maxGradients > MIN_ABS_GRAD_CREATE (:896) among the 4 pixels from i0
__device__ __forceinline__ int rndSelect4(const float* __restrict__ maxgrad, int i0, int w, int h, float minGrad, bool sel[4])
{
    int c = 0;
    const float4 g = *(const float4*)(maxgrad + i0);           // w % 16 == 0: the 4 pixels share a row
    const float gv[4] = { g.x, g.y, g.z, g.w };
    const int y = i0 / w, x0 = i0 - y * w;
    const bool row = y >= 1 && y <= h - 2;
    for (int k = 0; k < 4; k++) {
        sel[k] = row && x0 + k >= 1 && x0 + k <= w - 2 && gv[k] > minGrad;
        c += sel[k];
    }
    return c;
}

__global__ void __launch_bounds__(256) k_rnd_count(const float* __restrict__ maxgrad, int w, int h, float minGrad, int* __restrict__ tiles)
{
    __shared__ int sWarp[8];
    const int i0 = blockIdx.x * RND_TILE + 4 * threadIdx.x;
    bool sel[4];
    const int c = i0 < w * h ? rndSelect4(maxgrad, i0, w, h, minGrad, sel) : 0;
    int total;
    rndBlockScan<8>(c, sWarp, total);
    if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

// tiles[t] <- the first draw of tile t, tiles[nTiles] = out[0] = the number of draws N; the window after the last draw starts with
// the entry window's words that no draw replaces
__global__ void __launch_bounds__(1024) k_rnd_scan(int* __restrict__ tiles, int nTiles, RndEntry e, uint32_t* __restrict__ out)
{
    __shared__ int sWarp[32];
    int carry = 0;
    for (int base = 0; base < nTiles; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < nTiles ? tiles[i] : 0;
        int total;
        const int x = rndBlockScan<32>(v, sWarp, total);
        if (i < nTiles) tiles[i] = carry + x;
        carry += total;
    }
    if (threadIdx.x == 0) { tiles[nTiles] = carry; out[0] = (uint32_t)carry; }
    for (int m = threadIdx.x; m + carry < e.winLen; m += blockDim.x) out[1 + m] = e.W[m + carry];
}

// out[o] = sum_m rows[o * rowStride + m] * vecs[o * vecStride + m] over m < n, for o < nOut <= 64: four threads per output.
// out may alias vecs: every read is done before the first write.
__device__ __forceinline__ void rndBlockDots(const uint32_t* rows, int rowStride, const uint32_t* vecs, int vecStride, int n, int nOut,
                                             uint32_t* out)
{
    const int o = threadIdx.x >> 2, q = threadIdx.x & 3;
    uint32_t s = o < nOut ? rndDot(rows + o * rowStride, vecs + o * vecStride, n, q, 4) : 0u;
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    __syncthreads();
    if (o < nOut && q == 0) out[o] = s;
    __syncthreads();
}

__global__ void __launch_bounds__(256) k_rnd_fill(HypField cur, const float* __restrict__ maxgrad, int w, int h, const int* __restrict__ tiles,
                                                  const uint32_t* __restrict__ tab, RndEntry e, uint32_t* __restrict__ out)
{
    __shared__ uint32_t sW[RND_ROW], sExt[2 * RND_ROW], sVal[RND_TILE + RND_ROW];
    __shared__ int sWarp[8];
    const int n = w * h;
    const int i0 = blockIdx.x * RND_TILE + 4 * threadIdx.x;
    bool sel[4] = { false, false, false, false };
    const int c = i0 < n ? rndSelect4(maxgrad, i0, w, h, e.minGrad, sel) : 0;
    int total;
    int idx = rndBlockScan<8>(c, sWarp, total);
    const int s = tiles[blockIdx.x];                        // the tile's first draw
    const int N = tiles[gridDim.x];
    if (total > 0) {
        if (e.type == 0) {
            for (int j = threadIdx.x; j < total; j += blockDim.x) sVal[j] = rndLcgAt(e.W[0], (uint64_t)s + j + 1);
            __syncthreads();
        } else {
            const uint32_t* pw = tab + e.type * RND_TYPE_WORDS;
            const uint32_t* gen = pw + RND_POW_ROWS * RND_ROW;
            if (threadIdx.x < e.deg) sW[threadIdx.x] = e.W[threadIdx.x];
            __syncthreads();
            for (int b = 0; (s >> b) != 0; b++) {               // the window at draw s: one jump per set bit
                if (!((s >> b) & 1)) continue;
                if (threadIdx.x < e.deg) sExt[threadIdx.x] = sW[threadIdx.x];
                rndBlockDots(gen, RND_ROW, sW, 0, e.deg, e.deg - 1, sExt + e.deg);
                rndBlockDots(pw + b * RND_ROW, 0, sExt, 1, e.deg, e.deg, sW);
            }
            for (int q = 0; q < total; q += RND_ROW) {          // 64 draws at a time, then the window 64 draws later
                rndBlockDots(gen, RND_ROW, sW, 0, e.deg, RND_ROW, sVal + q);
                if (threadIdx.x < e.deg) sW[threadIdx.x] = sVal[q + RND_ROW - e.deg + threadIdx.x];
                __syncthreads();
            }
        }
    }
    if (i0 < n) {
        const int y = i0 / w, x0 = i0 - y * w;
        for (int k = 0; k < 4; k++) {
            const int i = i0 + k;
            if (y < 1 || y > h - 2 || x0 + k < 1 || x0 + k > w - 2) continue;   // border: untouched
            if (sel[k]) {                                       // DepthMapPixelHypothesis(idepth, idepth, VAR, VAR, 20), :898-903
                const float id = rndIdepth(rndOutput(e.type, sVal[idx++]));
                cur.hf[i] = make_float4(id, VAR_RANDOM_INIT_INITIAL, id, VAR_RANDOM_INIT_INITIAL);
                cur.hi[i] = make_int4(1, 0, 20, __float_as_int(0.f));
            } else {                                            // :907-908
                int4 hi = cur.hi[i];
                hi.x = 0; hi.y = 0;
                cur.hi[i] = hi;
            }
        }
    }
    for (int j = threadIdx.x; j < total; j += blockDim.x) {    // the last winLen draws are the window after the last draw
        const int m = s + j + e.winLen - N;
        if (m >= 0) out[1 + m] = sVal[j];
    }
}

static bool rndStateOk(const lsdgpu_rand_state* st)
{
    return st && st->type >= 0 && st->type < RND_TYPES && st->rear >= 0 && st->rear < rndWindowLen(st->type);
}

extern "C" int lsdgpu_rand_state_seed(int type, unsigned seed, lsdgpu_rand_state* st)
{   // __srandom_r, stdlib/random_r.c
    if (!st || type < 0 || type >= RND_TYPES) return -2;
    memset(st, 0, sizeof(*st));
    st->type = type;
    if (seed == 0) seed = 1;
    st->r[0] = seed;
    if (type == 0) return 0;
    const RndKind k = rndKind(type);
    int32_t word = (int32_t)seed;
    for (int i = 1; i < k.deg; i++) {                        // state[i] = (16807 * state[i - 1]) % 2147483647
        const long hi = word / 127773, lo = word % 127773;
        word = (int32_t)(16807 * lo - 2836 * hi);
        if (word < 0) word += 2147483647;
        st->r[i] = (uint32_t)word;
    }
    return lsdgpu_rand_state_advance(st, (int64_t)k.deg * 10, nullptr);
}

extern "C" int lsdgpu_rand_state_advance(lsdgpu_rand_state* st, int64_t n, int32_t* out)
{   // __random_r, stdlib/random_r.c, n times
    if (!rndStateOk(st) || n < 0) return -2;
    if (st->type == 0) {
        if (!out) { st->r[0] = rndLcgAt(st->r[0], (uint64_t)n); return 0; }
        for (int64_t i = 0; i < n; i++) out[i] = (int32_t)(st->r[0] = (st->r[0] * 1103515245u + 12345u) & 0x7fffffffu);
        return 0;
    }
    const RndKind k = rndKind(st->type);
    if (out) {
        int r = st->rear, f = (r + k.sep) % k.deg;
        for (int64_t i = 0; i < n; i++) {
            st->r[f] += st->r[r];
            out[i] = rndOutput(st->type, st->r[f]);
            if (++f == k.deg) f = 0;
            if (++r == k.deg) r = 0;
        }
        st->rear = r;
        return 0;
    }
    uint32_t W[RND_ROW];
    rndTableToWindow(st->type, st->rear, st->r, W);
    rndJumpWindow(st->type, W, (uint64_t)n);
    st->rear = (int)((st->rear + n) % k.deg);
    rndWindowToTable(st->type, st->rear, W, st->r);
    return 0;
}

extern "C" int lsdgpu_depth_init_random(lsdgpu_ctx* ctx, int kf_id, lsdgpu_rand_state* state, int64_t* n_draws)
{ LSD_LOCK(ctx);   // DepthMap::initializeRandomly :883-916
    if (!ctx) return -2;
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "initializeRandomly: unknown keyframe id");
    if (!rndStateOk(state)) return lsd_fail(ctx, "initializeRandomly: bad random state (type outside 0..4, or rear index outside its table)");
    if (!ctx->rndTabReady) {
        LSD_CHECK(ctx, cudaMemcpyAsync(ctx->rndTab, rndTables().w, sizeof(RndTables::w), cudaMemcpyHostToDevice, ctx->stream));
        ctx->rndTabReady = true;
    }
    RndEntry e;
    memset(&e, 0, sizeof(e));
    e.type = state->type; e.deg = rndKind(e.type).deg; e.winLen = rndWindowLen(e.type);
    e.minGrad = ctx->g.minUseGrad;
    rndTableToWindow(e.type, state->rear, state->r, e.W);
    const int n = ctx->w * ctx->h, nTiles = divUp(n, RND_TILE);
    k_rnd_count<<<nTiles, 256, 0, ctx->stream>>>(kf->maxgrad, ctx->w, ctx->h, e.minGrad, ctx->rndTiles);
    LAUNCH(ctx);
    k_rnd_scan<<<1, 1024, 0, ctx->stream>>>(ctx->rndTiles, nTiles, e, ctx->rndOut);
    LAUNCH(ctx);
    k_rnd_fill<<<nTiles, 256, 0, ctx->stream>>>(ctx->cur, kf->maxgrad, ctx->w, ctx->h, ctx->rndTiles, ctx->rndTab, e, ctx->rndOut);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    ctx->activeKf = kf_id; ctx->activeKfReactivated = false;       // :887-890
    int r = setDepthOnKeyframe(ctx, kf);                            // :915
    if (r) return r;
    uint32_t* res = (uint32_t*)ctx->hStageF;
    LSD_CHECK(ctx, cudaMemcpyAsync(res, ctx->rndOut, (1 + RND_ROW) * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    const int64_t draws = res[0];
    if (e.type != 0) state->rear = (int)((state->rear + draws) % e.deg);
    rndWindowToTable(e.type, state->rear, res + 1, state->r);
    if (n_draws) *n_draws = draws;
    return 0;
}

static int runRegularize(lsdgpu_ctx* ctx, bool removeOcclusions, int validityTH)
{
    DepthCam cam = depthCam(ctx);
    DepthGlobals G = depthGlobals(ctx);
    dim3 grid(divUp(cam.w, 32), divUp(cam.h, 8));
    std::swap(ctx->cur, ctx->oth);         // oth = previous current (the memcpy of :862), cur = output
    if (removeOcclusions) k_regularize<true><<<grid, 256, 0, ctx->stream>>>(ctx->oth, ctx->cur, cam, G, validityTH);
    else k_regularize<false><<<grid, 256, 0, ctx->stream>>>(ctx->oth, ctx->cur, cam, G, validityTH);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    return 0;
}
// regularizeDepthMapFillHoles() + regularizeDepthMap(false, TH) as one kernel (see k_fill_regularize); with
// setDepthOn != nullptr the kernel also does Frame::setDepth + the idepth pyramid of that keyframe
static int runFillRegularize(lsdgpu_ctx* ctx, int validityTH, FrameSlot* setDepthOn = nullptr)
{
    FrameSlot* kf = findSlot(ctx, ctx->activeKf);
    if (!kf) return lsd_fail(ctx, "no active keyframe");
    DepthCam cam = depthCam(ctx);
    DepthGlobals G = depthGlobals(ctx);
    const int grid = divUp(cam.w, FR_TW) * divUp(cam.h, FR_TH);
    std::swap(ctx->cur, ctx->oth);
    PyrPtrs id, var;
    for (int l = 0; l < LSD_LEVELS; l++) { id.l[l] = setDepthOn ? setDepthOn->idepth[l] : nullptr; var.l[l] = setDepthOn ? setDepthOn->idepthVar[l] : nullptr; }
    if (setDepthOn) {
        LSD_CHECK(ctx, launchPDL(k_fill_regularize<true>, dim3(grid), dim3(FR_THREADS), 0, ctx->stream, ctx->oth, ctx->cur, cam, G,
                                 (const float*)kf->maxgrad, validityTH, id, var, ctx->dScalars + 8, ctx->evCounter + 48, setDepthOn->dStats));
        setDepthOn->statsPending = true;
        setDepthOn->hasDepth = true; setDepthOn->idepthPyrValid = true;
        setDepthOn->depthHasBeenUpdatedFlag = true;                    // Frame.cpp:242
    } else
        LSD_CHECK(ctx, launchPDL(k_fill_regularize<false>, dim3(grid), dim3(FR_THREADS), 0, ctx->stream, ctx->oth, ctx->cur, cam, G,
                                 (const float*)kf->maxgrad, validityTH, id, var, (double*)nullptr, (unsigned int*)nullptr, (double*)nullptr));
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    return 0;
}

static int runFillHoles(lsdgpu_ctx* ctx)
{
    FrameSlot* kf = findSlot(ctx, ctx->activeKf);
    if (!kf) return lsd_fail(ctx, "no active keyframe");
    DepthCam cam = depthCam(ctx);
    DepthGlobals G = depthGlobals(ctx);
    dim3 grid(divUp(cam.w, 32), divUp(cam.h, 8));
    std::swap(ctx->cur, ctx->oth);
    k_fill_holes<<<grid, 256, 0, ctx->stream>>>(ctx->oth, ctx->cur, cam, G, kf->maxgrad);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    return 0;
}

// the hypotheses of keyframe kf from a 16-byte aligned device AoS (the staging buffer or a caller's), then the optional
// re-activation regularization and setDepth
static int setHypotheses(lsdgpu_ctx* ctx, int kf_id, FrameSlot* kf, const lsdgpu_hyp* daos, int reactivated, int do_set_depth)
{
    const int n = ctx->w * ctx->h;
    k_hyp_from_aos<<<divUp(n, 256), 256, 0, ctx->stream>>>(daos, ctx->cur, n);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    ctx->activeKf = kf_id; ctx->activeKfReactivated = reactivated != 0;
    if (reactivated) {
        kf->numMappedOnThis = 0; kf->numFramesTrackedOnThis = 0;                   // :932-933
        int r = runRegularize(ctx, false, VAL_SUM_MIN_FOR_KEEP);                   // :961
        if (r) return r;
    }
    if (do_set_depth) return setDepthOnKeyframe(ctx, kf);
    return 0;
}

extern "C" int lsdgpu_depth_set_hypotheses(lsdgpu_ctx* ctx, int kf_id, const lsdgpu_hyp* aos, int reactivated, int do_set_depth)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "unknown keyframe id");
    const int n = ctx->w * ctx->h;
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(ctx->hStageF, aos, (size_t)n * 32);
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->dStageF, ctx->hStageF, (size_t)n * 32, cudaMemcpyHostToDevice, ctx->stream));
    return setHypotheses(ctx, kf_id, kf, (const lsdgpu_hyp*)ctx->dStageF, reactivated, do_set_depth);
}

extern "C" int lsdgpu_depth_set_hypotheses_device(lsdgpu_ctx* ctx, int kf_id, const lsdgpu_hyp* d_aos, int reactivated,
                                                  int do_set_depth, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "unknown keyframe id");
    int r = checkDevicePtr(ctx, "depth_set_hypotheses_device", "the hypotheses", d_aos, 16);
    if (r) return r;
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    if ((r = setHypotheses(ctx, kf_id, kf, d_aos, reactivated, do_set_depth))) return r;
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    return 0;
}

extern "C" int lsdgpu_depth_download(lsdgpu_ctx* ctx, lsdgpu_hyp* aos_out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    const int n = ctx->w * ctx->h;
    k_hyp_to_aos<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->cur, (lsdgpu_hyp*)ctx->dStageF, n);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    LSD_CHECK(ctx, cudaMemcpyAsync(aos_out, ctx->dStageF, (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int lsdgpu_depth_download_device(lsdgpu_ctx* ctx, lsdgpu_hyp* d_aos, size_t capacity, void* stream)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    const int n = ctx->w * ctx->h;
    int r = checkCapacity(ctx, "depth_download_device", "the depth map", (size_t)n * sizeof(lsdgpu_hyp), capacity);
    if (r || (r = checkDevicePtr(ctx, "depth_download_device", "the output", d_aos, 16))) return r;
    LSD_CHECK(ctx, afterCallerStream(ctx, stream));
    k_hyp_to_aos<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->cur, d_aos, n);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    LSD_CHECK(ctx, beforeCallerStream(ctx, stream));
    return 0;
}

extern "C" int lsdgpu_depth_download_integral(lsdgpu_ctx* ctx, int32_t* out)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    k_integral_rows<<<divUp(ctx->h, 64), 64, 0, ctx->stream>>>(ctx->cur, ctx->integral, ctx->w, ctx->h);
    LAUNCH(ctx);
    k_integral_cols<<<divUp(ctx->w, 64), 64, 0, ctx->stream>>>(ctx->integral, ctx->w, ctx->h);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    LSD_CHECK(ctx, cudaMemcpyAsync(out, ctx->integral, (size_t)ctx->w * ctx->h * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

static void prepareForStereoWith(const lsdgpu_ctx* ctx, const FrameSlot* fr, RefConst& rc)
{
    prepareStereoConsts(ctx->cam[0].K, fr->thisToParent, fr->thisToParent + 4, fr->thisToParent[7], rc);
}

static int setupObserve(lsdgpu_ctx* ctx, const lsdgpu_ref_desc* refs, int n_refs, FrameSlot* kf)
{   // DepthMap.cpp:1079-1105
    if (n_refs <= 0 || n_refs > LSD_MAX_REFS) return lsd_fail(ctx, "bad number of reference frames");
    ObserveParams& OP = ctx->hObs;
    OP.nRefs = n_refs;
    OP.byIdSize = 0;
    for (int k = 0; k < n_refs; k++) {
        FrameSlot* fr = findSlot(ctx, refs[k].frame_id);
        if (!fr) return failMissing(ctx, refs[k].frame_id, "unknown reference frame id");
        RefConst& rc = OP.refs[k];
        if (refs[k].tracked_on_kf) {
            // :1096-1097 refToKf = frame->pose->thisToParent_raw
            if (fr->parentId != kf->id) return lsd_fail(ctx, "reference frame declared tracked_on_kf but its tracking parent is not the active keyframe");
            prepareForStereoWith(ctx, fr, rc);
        } else {
            // :1098-1099 refToKf = activeKeyFrame->getScaledCamToWorld().inverse() * frame->getScaledCamToWorld(): the absolute
            // poses live in the caller's pose graph (FramePoseStruct / KeyFrameGraph), so the caller hands the product over
            const double* q = refs[k].refToKf_qts;
            const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
            if (!(n2 > 0.25 && n2 < 4.0) || !(q[7] > 0)) return lsd_fail(ctx, "reference frame not tracked on the active keyframe: refToKf_qts must hold a unit quaternion and a positive scale");
            prepareStereoConsts(ctx->cam[0].K, q, q + 4, q[7], rc);
        }
        rc.initialTrackedResidual = fr->initialTrackedResidual;
        rc.id = fr->id;
        rc.trackedOnActive = refs[k].tracked_on_kf ? 1 : 0;       // gate of the tracking mask, DepthMap.cpp:245 / :322
        rc.image = fr->image[0];
        rc.goodMask = fr->hasGoodMask ? fr->goodMask : nullptr;
        if (k == 0) OP.byIdOffset = fr->id;
        while (OP.byIdSize + OP.byIdOffset <= fr->id) {
            if (OP.byIdSize >= LSD_MAX_ID_SPAN) return lsd_fail(ctx, "reference id span too large");
            OP.byId[OP.byIdSize++] = k;
        }
    }
    OP.oldestIdx = 0; OP.newestIdx = n_refs - 1;
    OP.reactivated = ctx->activeKfReactivated ? 1 : 0;
    OP.kfNumTracked = kf->numFramesTrackedOnThis; OP.kfNumMapped = kf->numMappedOnThis;
    return 0;
}

// ids only: every frame was tracked on the active keyframe (the common case, SlamSystem.cpp:559-575)
static int setupObserve(lsdgpu_ctx* ctx, const int* ref_ids, int n_refs, FrameSlot* kf)
{
    if (n_refs <= 0 || n_refs > LSD_MAX_REFS) return lsd_fail(ctx, "bad number of reference frames");
    lsdgpu_ref_desc d[LSD_MAX_REFS];
    memset(d, 0, sizeof(d));
    for (int k = 0; k < n_refs; k++) {
        d[k].frame_id = ref_ids[k]; d[k].tracked_on_kf = 1;
        const FrameSlot* fr = findSlot(ctx, ref_ids[k]);
        if (fr && fr->parentId != kf->id)
            return lsd_fail(ctx, "reference frame was not tracked on the active keyframe: pass its refToKf through lsdgpu_depth_update_keyframe_refs");
    }
    return setupObserve(ctx, d, n_refs, kf);
}

static int runObserve(lsdgpu_ctx* ctx, const int* ref_ids, int n_refs, bool hostParamsReady = false)
{
    FrameSlot* kf = findSlot(ctx, ctx->activeKf);
    if (!kf) return lsd_fail(ctx, "no active keyframe");
    if (!hostParamsReady) {
        int r = setupObserve(ctx, ref_ids, n_refs, kf);
        if (r) return r;
    }
    DepthCam cam = depthCam(ctx);
    DepthGlobals G = depthGlobals(ctx);
    const int grid = divUp((cam.w - 6) * (cam.h - 6), OBS_PIX_PER_CTA);
    LSD_CHECK(ctx, launchPDL(k_observe, dim3(grid), dim3(OBS_THREADS), 0, ctx->stream, ctx->cur, cam, G, (const float*)kf->image[0],
                             (const float4*)kf->grad[0], (const float*)kf->maxgrad, ctx->hObs));
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    return 0;
}

extern "C" int lsdgpu_depth_observe(lsdgpu_ctx* ctx, const int* ref_ids, int n_refs)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    return runObserve(ctx, ref_ids, n_refs);
}
extern "C" int lsdgpu_depth_regularize_fill_holes(lsdgpu_ctx* ctx)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    return runFillHoles(ctx);
}
extern "C" int lsdgpu_depth_regularize(lsdgpu_ctx* ctx, int removeOcclusions, int validityTH)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    return runRegularize(ctx, removeOcclusions != 0, validityTH);
}

extern "C" int lsdgpu_depth_update_keyframe(lsdgpu_ctx* ctx, const int* ref_ids, int n_refs)
{ LSD_LOCK(ctx);   // DepthMap::updateKeyframe :1072-1213
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, ctx->activeKf);
    if (!kf) return lsd_fail(ctx, "updateKeyframe: depth map is not valid (no active keyframe)");
    int r = runObserve(ctx, ref_ids, n_refs);                      // :1127
    if (r) return r;
    r = runFillRegularize(ctx, VAL_SUM_MIN_FOR_KEEP,               // :1135 + :1143 (+ setDepth :1150-1157 in the same kernel)
                          kf->depthHasBeenUpdatedFlag ? nullptr : kf);
    if (r) return r;
    kf->numMappedOnThis++;                                         // :1165
    return 0;
}

extern "C" int lsdgpu_depth_update_keyframe_refs(lsdgpu_ctx* ctx, const lsdgpu_ref_desc* refs, int n_refs)
{ LSD_LOCK(ctx);   // DepthMap::updateKeyframe :1072-1213 with the reference-frame set-up of :1085-1101 spelled out by the caller
    if (!ctx || !refs) return lsd_fail(ctx, "update_keyframe_refs: null argument");
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, ctx->activeKf);
    if (!kf) return lsd_fail(ctx, "updateKeyframe: depth map is not valid (no active keyframe)");
    int r = setupObserve(ctx, refs, n_refs, kf);
    if (r) return r;
    r = runObserve(ctx, nullptr, n_refs, true);                    // :1127 (parameters already in ctx->hObs)
    if (r) return r;
    r = runFillRegularize(ctx, VAL_SUM_MIN_FOR_KEEP, kf->depthHasBeenUpdatedFlag ? nullptr : kf);
    if (r) return r;
    kf->numMappedOnThis++;                                         // :1165
    return 0;
}

static int runPropagate(lsdgpu_ctx* ctx, FrameSlot* kf, FrameSlot* nk)
{   // DepthMap::propagateDepth :475-653
    const int n = ctx->w * ctx->h;
    lsd::SE3<double> tp;
    for (int i = 0; i < 4; i++) tp.q[i] = nk->thisToParent[i];
    for (int i = 0; i < 3; i++) tp.t[i] = nk->thisToParent[4 + i];
    lsd::quatNormalize(tp.q);                                      // se3FromSim3: SE3(quaternion, translation)
    lsd::SE3<double> oldToNew = lsd::se3Inverse(tp);               // :503
    double Rd[9];
    lsd::quatToMatrix(oldToNew.q, Rd);
    PropParams P;
    for (int i = 0; i < 9; i++) P.R[i] = (float)Rd[i];
    for (int i = 0; i < 3; i++) P.t[i] = (float)oldToNew.t[i];
    P.trackingWasGood = (nk->parentId == kf->id && nk->hasGoodMask) ? nk->goodMask : nullptr;      // :508
    P.activeKFImage = kf->image[0];
    P.newKFMaxGrad = nk->maxgrad;
    P.newKFImage = nk->image[0];
    LSD_CHECK(ctx, cudaMemsetAsync(ctx->propHead, 0xff, (size_t)n * 4, ctx->stream));
    DepthCam cam = depthCam(ctx);
    DepthGlobals G = depthGlobals(ctx);
    k_prop_project<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->cur, cam, G, P, ctx->propHead, ctx->propNext, ctx->propVal);
    LAUNCH(ctx);
    k_prop_resolve<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->oth, n, ctx->propHead, ctx->propNext, ctx->propVal);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    std::swap(ctx->cur, ctx->oth);                                 // :637
    return 0;
}

extern "C" int lsdgpu_depth_propagate(lsdgpu_ctx* ctx, int new_kf_id)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, ctx->activeKf);
    FrameSlot* nk = findSlot(ctx, new_kf_id);
    if (!kf || !nk) return failMissing(ctx, new_kf_id, "propagateDepth: unknown keyframe");
    return runPropagate(ctx, kf, nk);
}

extern "C" int lsdgpu_depth_create_keyframe(lsdgpu_ctx* ctx, int new_kf_id, double new_qts[8])
{ LSD_LOCK(ctx);   // DepthMap::createKeyFrame :1222-1327
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, ctx->activeKf);
    FrameSlot* nk = findSlot(ctx, new_kf_id);
    if (!kf) return lsd_fail(ctx, "createKeyFrame: depth map is not valid");
    if (!nk) return failMissing(ctx, new_kf_id, "createKeyFrame: unknown new keyframe");
    if (nk->parentId < 0) return lsd_fail(ctx, "createKeyFrame: new keyframe has no tracking parent");
    lsd::SE3<double> tp;
    for (int i = 0; i < 4; i++) tp.q[i] = nk->thisToParent[i];
    for (int i = 0; i < 3; i++) tp.t[i] = nk->thisToParent[4 + i];
    lsd::quatNormalize(tp.q);
    lsd::SE3<double> oldToNew = lsd::se3Inverse(tp);               // :1246
    int r = runPropagate(ctx, kf, nk);                             // :1250
    if (r) return r;
    ctx->activeKf = new_kf_id; ctx->activeKfReactivated = false;   // :1255-1258
    r = runRegularize(ctx, true, VAL_SUM_MIN_FOR_KEEP);            // :1263
    if (r) return r;
    r = runFillRegularize(ctx, VAL_SUM_MIN_FOR_KEEP);              // :1270 + :1277
    if (r) return r;
    const int n = ctx->w * ctx->h;
    const int nb = divUp(n, 256);
    // :1286-1294: the reference's sequential `float +=` over the valid hypotheses, reproduced bit for bit (seqsum.cuh)
    const int seqRuns = divUp(n, SEQ_RUN);
    k_seqsum_table<<<divUp(seqRuns, 8), 256, 0, ctx->stream>>>(ctx->cur.hf, ctx->cur.hi, n, seqRuns, ctx->seqTable, ctx->seqFlags, ctx->seqCounts);
    LAUNCH(ctx);
    k_seqsum_walk<<<1, 32, 0, ctx->stream>>>(ctx->cur.hf, ctx->cur.hi, n, seqRuns, ctx->seqTable, ctx->seqFlags, ctx->seqCounts, ctx->dScalars);
    LAUNCH(ctx);
    k_rescale<<<nb, 256, 0, ctx->stream>>>(ctx->cur, n, ctx->dScalars);                          // :1295-1304
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    LSD_CHECK(ctx, cudaMemcpyAsync(ctx->hScalars + 4, ctx->dScalars, 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    const float rescaleFactor = (float)ctx->hScalars[4 + 2];
    lsd::SE3<double> back = lsd::se3Inverse(oldToNew);             // :1305 sim3FromSE3(oldToNew_SE3.inverse(), rescaleFactor)
    for (int i = 0; i < 4; i++) nk->thisToParent[i] = back.q[i];
    for (int i = 0; i < 3; i++) nk->thisToParent[4 + i] = back.t[i];
    nk->thisToParent[7] = rescaleFactor;
    if (new_qts) memcpy(new_qts, nk->thisToParent, sizeof(nk->thisToParent));
    return setDepthOnKeyframe(ctx, nk);                            // :1311
}

__global__ void k_seqsum_pack(const float* __restrict__ x, const unsigned char* __restrict__ valid, int n, float4* hf, int4* hi)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    hf[i] = make_float4(0.f, 0.f, x[i], 0.f);
    hi[i] = make_int4(valid ? (valid[i] != 0) : 1, 0, 0, 0);
}

// The sequential `float sum = 0; for (i) if (valid[i]) sum += x[i];` of DepthMap.cpp:1286-1293 on arbitrary host data, through
// the kernels createKeyFrame uses (seqsum.cuh) -- exposed so the bit-exactness of that reproduction can be tested on adversarial
// inputs (ties, binade crossings, negative / non-finite terms), which real depth maps rarely contain.
extern "C" int lsdgpu_seq_sum_f32(lsdgpu_ctx* ctx, const float* x, const unsigned char* valid, int n, float* sum, int* count)
{ LSD_LOCK(ctx);
    if (!ctx || !x || n < 0 || !sum) return lsd_fail(ctx, "seq_sum_f32: bad arguments");
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    if (n == 0) { *sum = 0.f; if (count) *count = 0; return 0; }
    const int runs = divUp(n, SEQ_RUN);
    char* buf = nullptr;
    const size_t bx = alignUp((size_t)n * 4, 256), bv = alignUp((size_t)n, 256), bf = alignUp((size_t)n * 16, 256),
                 bt = alignUp((size_t)runs * SEQ_NBIN * sizeof(int2), 256), bg = alignUp((size_t)runs, 256), bc = alignUp((size_t)runs * 4, 256);
    LSD_CHECK(ctx, cudaMalloc((void**)&buf, bx + bv + 2 * bf + bt + bg + bc + 256));
    char* p = buf;
    float* dx = (float*)p; p += bx;
    unsigned char* dv = (unsigned char*)p; p += bv;
    float4* hf = (float4*)p; p += bf;
    int4* hi = (int4*)p; p += bf;
    int2* table = (int2*)p; p += bt;
    unsigned char* flags = (unsigned char*)p; p += bg;
    int* counts = (int*)p; p += bc;
    double* out = (double*)p;
    int rc = 0;
    do {
        if (cudaMemcpyAsync(dx, x, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) { rc = 1; break; }
        if (valid && cudaMemcpyAsync(dv, valid, (size_t)n, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) { rc = 1; break; }
        k_seqsum_pack<<<divUp(n, 256), 256, 0, ctx->stream>>>(dx, valid ? dv : nullptr, n, hf, hi);
        k_seqsum_table<<<divUp(runs, 8), 256, 0, ctx->stream>>>(hf, hi, n, runs, table, flags, counts);
        k_seqsum_walk<<<1, 32, 0, ctx->stream>>>(hf, hi, n, runs, table, flags, counts, out);
        double h[3];
        if (cudaMemcpyAsync(h, out, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) { rc = 1; break; }
        if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) { rc = 1; break; }
        *sum = (float)h[0];
        if (count) *count = (int)h[1];
    } while (0);
    cudaFree(buf);
    if (rc) return lsd_fail(ctx, "seq_sum_f32: CUDA error");
    return 0;
}

// Frame::takeReActivationData(currentDepthMap), Frame.cpp:107-145.  The pool buffers of a fresh Frame are defined as
// zero-filled (SURVEY appendix A.12); later takes of the same frame keep the entries of invalid pixels, as the reference does.
static int takeReactivationData(lsdgpu_ctx* ctx, FrameSlot* kf)
{
    const int n = ctx->w * ctx->h;
    if (!kf->reactAllocated) {
        LSD_CHECK(ctx, cudaMemsetAsync(kf->reactIdepth, 0, (size_t)n * 4, ctx->stream));
        LSD_CHECK(ctx, cudaMemsetAsync(kf->reactVar, 0, (size_t)n * 4, ctx->stream));
        LSD_CHECK(ctx, cudaMemsetAsync(kf->reactValidity, 0, (size_t)n, ctx->stream));
        kf->reactAllocated = true;
    }
    k_take_reactivation<<<divUp(n, 256), 256, 0, ctx->stream>>>(ctx->cur, kf->reactIdepth, kf->reactVar, kf->reactValidity, n);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    kf->reactValid = true;
    return 0;
}

extern "C" int lsdgpu_depth_finalize_keyframe(lsdgpu_ctx* ctx)
{ LSD_LOCK(ctx);   // DepthMap::finalizeKeyFrame :1363-1395
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, ctx->activeKf);
    if (!kf) return lsd_fail(ctx, "finalizeKeyFrame: depth map is not valid");
    int r = runFillRegularize(ctx, VAL_SUM_MIN_FOR_KEEP, kf);            // :1373 + :1379 + setDepth :1385
    if (r) return r;
    return takeReactivationData(ctx, kf);                                // :1387 (calculateMeanInformation :1386 returns at once, Frame.cpp:178)
}

extern "C" int lsdgpu_frame_take_reactivation_data(lsdgpu_ctx* ctx, int kf_id)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "unknown keyframe id");
    if (ctx->activeKf != kf_id) return lsd_fail(ctx, "takeReActivationData: the keyframe is not the active one");
    return takeReactivationData(ctx, kf);
}

extern "C" int lsdgpu_frame_download_reactivation_data(lsdgpu_ctx* ctx, int kf_id, float* idepth_reAct, float* idepthVar_reAct, uint8_t* validity_reAct)
{ LSD_LOCK(ctx);
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findFrame(ctx, kf_id);                                 // a minimized keyframe: from its record
    if (!kf) return lsd_fail(ctx, "unknown keyframe id");
    if (!kf->reactValid) return lsd_fail(ctx, "keyframe has no reactivation data");
    const size_t n = (size_t)ctx->w * ctx->h;
    // from an offloaded keyframe's host body the copies are host to host, which cudaMemcpyAsync need not order behind the stream
    if (kf->record[TIER_HOST]) LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    if (idepth_reAct) LSD_CHECK(ctx, cudaMemcpyAsync(idepth_reAct, kf->reactIdepth, n * 4, cudaMemcpyDefault, ctx->stream));
    if (idepthVar_reAct) LSD_CHECK(ctx, cudaMemcpyAsync(idepthVar_reAct, kf->reactVar, n * 4, cudaMemcpyDefault, ctx->stream));
    if (validity_reAct) LSD_CHECK(ctx, cudaMemcpyAsync(validity_reAct, kf->reactValidity, n, cudaMemcpyDefault, ctx->stream));
    LSD_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int lsdgpu_depth_set_from_existing_kf(lsdgpu_ctx* ctx, int kf_id)
{ LSD_LOCK(ctx);   // DepthMap::setFromExistingKF :920-962
    LSD_CHECK(ctx, cudaSetDevice(ctx->device));
    FrameSlot* kf = findSlot(ctx, kf_id);
    if (!kf) return failMissing(ctx, kf_id, "unknown keyframe id");
    if (!kf->hasDepth) return lsd_fail(ctx, "setFromExistingKF: keyframe has no depth");          // assert(kf->hasIDepthBeenSet()), :922
    if (!kf->reactValid) return lsd_fail(ctx, "setFromExistingKF: keyframe has no reactivation data");
    const int n = ctx->w * ctx->h;
    k_set_from_existing<<<divUp(n, 256), 256, 0, ctx->stream>>>(kf->reactIdepth, kf->reactVar, kf->reactValidity, ctx->cur, n);
    LAUNCH(ctx);
    LSD_CHECK(ctx, cudaGetLastError());
    ctx->activeKf = kf_id; ctx->activeKfReactivated = true;                                       // :925, :935
    kf->numMappedOnThis = 0; kf->numFramesTrackedOnThis = 0;                                      // :932-933
    return runRegularize(ctx, false, VAL_SUM_MIN_FOR_KEEP);                                       // :961
}
